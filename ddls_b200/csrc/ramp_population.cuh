// ramp_population.cuh -- K independent PPO, IMPALA or PG trainings of the GNN policy in one environment batch (include/ramp_b200.h:
// ramp_population_*).  Included by ramp_policy.cu after the learner.
//
// The environment's B = K b episodes are K contiguous groups of b; group k acts with weight set k and learns only from its own
// episodes with its own config.  The sets may differ in shape: set k has its own ramp_policy_config_t, and the kernels that depend
// on it take set k's entry of the device table d_sets (PopSet: its PolicyDev with `w` at its weights, and its slices of the ragged
// buffers).  Every kernel here runs the statements of the single policy's kernel (the shared *_body functions of ramp_policy.cu /
// ramp_policy_learn.cuh) on one set's slice, with the set taken from the launch:
//
//   ramp_pop_embed_grad_kernel   persistent CTAs over (set, job type) items, grid-strided past the resident CTAs: the MeanPool
//                                rounds (forward: states kept, embeddings [K][n_models][out_node]) or their backward
//   ramp_pop_head_kernel         blockIdx.y = set: the read-out of the set's episodes / rows, its weights staged per CTA
//   ramp_pop_gae_kernel          one 1,024-thread CTA per group: GAE (PG: discounted returns) over the group's columns of the
//                                [T][B] trajectory, its live rows t-major into the group's slice of the train batch,
//                                standardised with the group's mean / std when asked
//   ramp_pop_head_grad_kernel    blockIdx.y = set, one warp per launch row: the rows of every group's minibatch / SGD step in one
//                                launch
//   ramp_pop_head_reduce_kernel  one thread per (set, read-out weight): the sum over the set's rows in row order
//   ramp_pop_finish_kernel / ramp_pop_adam_kernel   blockIdx.y = set: the job types' sum, the norm partials, clip and Adam
//   ramp_pop_learn_stats_kernel  one thread per set: the last pass's means and update_kl
//   ramp_pop_impala_batch_kernel one thread per (set, fragment row): IMPALA's fragments of the group's columns
//   ramp_pop_vtrace_kernel       one warp per (set, fragment): V-trace with the set's gamma and clip thresholds
//   ramp_pop_impala_*_stats_kernel, ramp_pop_pg_stats_kernel   one thread per set: its statistics
//
// So group k computes what one policy with set k's weights computes on a b-episode environment with the same episode streams, bit
// for bit: no float atomics, and every reduction in the single kernel's order.
#pragma once

namespace ramp {

// set s of a population: its configuration's layout with `w` at its own weights -- the PolicyDev the single policy's kernels take
// -- and where its slices of the population's ragged buffers start.  Kernels serving one set per CTA stage the entry in shared
// memory (pop_stage_set) and run the bodies on it.
struct PopSet {
    PolicyDev P;
    int64_t n_w, w_off;                   // weights; their offset in every [sum n_w] buffer (weights, gradient, Adam's m / v)
    int64_t n_gnn, gpart_off;             // the rounds' weights; set s's [n_models][n_gnn] job-type partials
    int64_t emb_off;                      // set s's [n_models][out_node] embeddings
};

// sets[s] into shared `dst` by the whole CTA, word by word (the caller syncs before `dst` is rewritten)
__device__ __forceinline__ void pop_stage_set(const PopSet* sets, int s, PopSet* dst) {
    const int32_t* src = reinterpret_cast<const int32_t*>(sets + s);
    int32_t* d = reinterpret_cast<int32_t*>(dst);
    for (int i = threadIdx.x; i < (int)(sizeof(PopSet) / 4); i += blockDim.x) d[i] = src[i];
    __syncthreads();
}

struct PopHead {
    int32_t per;                          // episodes / rows of one set
    int32_t stride;                       // rows from one set's first to the next's (per, or a set's whole batch when the launch
                                          // covers a slice of it)
    const unsigned long long* seeds;      // [K] the sets' act seeds (sample), mixed with `mix` as ramp_policy_act mixes its call count
    unsigned long long mix;
};

// dynamic shared memory: the largest set's read-out staging.  The set's configuration is read from shared memory, not the constant
// bank as in ramp_policy_head_kernel, and needs about 30 more registers: at 80 (three CTAs per SM) ptxas spills about 900 bytes
__global__ void __launch_bounds__(256, 2) ramp_pop_head_kernel(const PopSet* sets, const HeadArgs base, const PopHead ph) {
    __shared__ PopSet S;
    const int s = blockIdx.y;
    pop_stage_set(sets, s, &S);
    const size_t o = (size_t)s * ph.stride, A = S.P.c.n_actions;
    HeadArgs a = base;
    a.n = ph.per;
    a.model += o; a.mask += o * A; a.actions += o;
    if (a.obs_dyn) a.obs_dyn += o * 11;
    if (a.graph_features) a.graph_features += o * S.P.c.in_features_graph;
    if (a.done) a.done += o;
    if (a.logits) a.logits += o * A;
    if (a.value) a.value += o;
    if (a.logp) a.logp += o;
    a.emb += S.emb_off;
    if (a.sample) a.seed = ph.seeds[s] ^ ph.mix;
    head_body(S.P, S.P.w, a, blockIdx.x, gridDim.x);
}

struct PopEmbed {
    int32_t K, n_models;
    int32_t rec_stride;                   // backward: floats per head record of the launch (the largest set's)
};

// item = set n_models + job type; the forward's n_rows / emb and the backward's records and partials are the set's slices
template <int MODE>
__global__ void __launch_bounds__(256, 1) ramp_pop_embed_grad_kernel(const PopSet* sets, const ModelDev* models, const GradModelDev* gms,
                                                                     const EmbGradArgs g, const PopEmbed pe) {
    __shared__ PopSet S;
    const int nm = pe.n_models;
    for (int item = blockIdx.x; item < pe.K * nm; item += gridDim.x) {
        const int s = item / nm, m = item - s * nm;
        pop_stage_set(sets, s, &S);
        EmbGradArgs e = g;
        if (MODE == EMB_FORWARD) {
            if (e.n_rows) e.n_rows += s;
            if (e.emb) e.emb += S.emb_off;
        } else {
            e.rec += (size_t)s * e.rows * pe.rec_stride;
            e.row_model += (size_t)s * e.rows;
            e.gpart += S.gpart_off;
            e.n_gnn = S.n_gnn;
        }
        embed_grad_body<MODE>(S.P, S.P.w, models, gms + (size_t)s * nm, e, m);
        __syncthreads();                  // the next item reuses the shared staging
    }
}

__global__ void __launch_bounds__(1024) ramp_pop_gae_kernel(const GaeArgs* sets, int32_t ld) {
    const GaeArgs a = sets[blockIdx.x];
    gae_body(a, ld);
}

// blockIdx.y = set: args[k] is group k's GradArgs for a minibatch starting at 0 (records, row model and statistics already at k mb);
// keys: the pass's [K]
__global__ void __launch_bounds__(256) ramp_pop_head_grad_kernel(const PopSet* sets, const GradArgs* args, int32_t start,
                                                                 const unsigned long long* keys, int32_t first_pass) {
    __shared__ PopSet S;
    __shared__ GradArgs g;                // in shared memory too: in registers beside the set's fields it spills
    const int s = blockIdx.y;
    if (threadIdx.x == 0) {
        g = args[s];
        g.start = start; g.key = keys[s];
        if (!first_pass) g.logp_old = nullptr;
    }
    pop_stage_set(sets, s, &S);
    head_grad_body(S.P, S.P.w, g, blockIdx.x * LRN_WARPS + (threadIdx.x >> 5));
}

// ramp_policy_head_reduce_kernel over every set: one thread per (set, read-out weight).  segs: [K][HEAD_SEGS] set s's segments on
// its own records, their blob offsets into the population's weights `w`; n_segs: [K]; first: [K] set s's first thread
__global__ void __launch_bounds__(256) ramp_pop_head_reduce_kernel(const Seg* segs, const int32_t* n_segs, const int64_t* first, int32_t K,
                                                                   int64_t total, const float* w, float* grad) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        int s = 0, hi = K - 1;
        while (s < hi) {                                            // the last set starting at or before e
            const int mid = (s + hi + 1) >> 1;
            if (first[mid] <= e) s = mid; else hi = mid - 1;
        }
        const Seg* ss = segs + (size_t)s * HEAD_SEGS;
        const int n = n_segs[s];
        int si = 0;
        int64_t off = e - first[s];
        while (si + 1 < n && off >= seg_size(ss[si])) { off -= seg_size(ss[si]); ++si; }
        grad[ss[si].w + off] = seg_element(ss[si], off, w);
    }
}

__global__ void __launch_bounds__(256) ramp_pop_finish_kernel(const PopSet* sets, const float* gpart, int32_t n_models, float* grad, double* norm_part) {
    const size_t s = blockIdx.y;
    const PopSet& S = sets[s];
    grad_finish_body(gpart + S.gpart_off, n_models, S.n_gnn, S.n_w, grad + S.w_off, norm_part + s * LRN_GRID);
}

// args[k]: group k's AdamArgs for minibatch 0 of a pass; minibatch j starts at `start` and writes its statistics j rows further
__global__ void __launch_bounds__(256) ramp_pop_adam_kernel(const PopSet* sets, const AdamArgs* args, int32_t start, int32_t j, int32_t parity) {
    AdamArgs a = args[blockIdx.y];
    a.start = start; a.parity = parity; a.stats += (size_t)j * RAMP_PPO_STATS_LEN;
    adam_body(a, sets[blockIdx.y].n_w);
}

// kl: [K][2] the sets' kl_coeff and kl_target
__global__ void ramp_pop_learn_stats_kernel(const double* mb_stats, int32_t n_mb, int32_t n_mb_used, const float* kl, const int32_t* n_rows,
                                            double* out, int32_t K) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= K) return;
    learn_stats_body(mb_stats + (size_t)s * n_mb * RAMP_PPO_STATS_LEN, n_mb_used, kl[2 * s], kl[2 * s + 1], n_rows + s,
                     out + (size_t)s * RAMP_PPO_STATS_LEN);
}

// ---- IMPALA and PG: the single learner's bodies on one set's slices ----

// IMPALA's fragment rows of every group, one thread per (set, row): a is set 0's (its a.B = b episodes per group), set s reads
// the columns [s b, (s + 1) b) of the [T][K b] trajectory and writes its T b rows s T b rows further
__global__ void ramp_pop_impala_batch_kernel(const ImpalaBatchArgs base, int32_t K) {
    const int64_t R = (int64_t)base.T * base.B;
    const int64_t gi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (gi >= K * R) return;
    const int64_t s = gi / R;
    const size_t col = (size_t)s * base.B, o = (size_t)s * R, A = base.A;
    ImpalaBatchArgs a = base;
    a.t_obs += col * 11; a.t_model += col; a.t_mask += col * A; a.t_action += col; a.t_logp += col; a.t_reward += col; a.t_done += col;
    a.obs += o * 11; a.model += o; a.mask += o * A; a.action += o; a.blogp += o; a.reward += o; a.done += o; a.n_rows += s;
    impala_batch_body(a, gi - s * R, K * base.B);
}

// one warp per (set, fragment): sets[k] is set k's VtraceArgs (its gamma, clip thresholds and row slices); the step's fragments
// and first row are the launch's
__global__ void __launch_bounds__(256) ramp_pop_vtrace_kernel(const VtraceArgs* sets, int32_t K, int32_t n_frag, int32_t row0) {
    const int gi = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (gi >= K * n_frag) return;
    const int s = gi / n_frag;
    VtraceArgs a = sets[s];
    a.n_frag = n_frag; a.row0 = row0;
    vtrace_body(a, gi - s * n_frag, threadIdx.x & 31);
}

// one thread per set: SGD step k (of n_sgd) of every set, whose launch rows are mb apart and whose fragment rows R apart; coef:
// [K][2] the sets' vf_loss_coeff and entropy_coeff
__global__ void ramp_pop_impala_step_stats_kernel(const float* row_stats, const int32_t* row_model, int32_t mb, int32_t row0, const float* log_rho,
                                                  int32_t R, const double* coef, const double* norm_part, double* step_stats, int32_t n_sgd,
                                                  int32_t k, int32_t K) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= K) return;
    impala_step_stats_body(row_stats + (size_t)s * mb * RS_N, row_model + (size_t)s * mb, mb, row0, log_rho + (size_t)s * R, coef[2 * s],
                           coef[2 * s + 1], norm_part + (size_t)s * LRN_GRID, step_stats + ((size_t)s * n_sgd + k) * RAMP_IMPALA_STATS_LEN);
}

__global__ void ramp_pop_impala_learn_stats_kernel(const double* step_stats, int32_t n_sgd, double* out, int32_t K) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= K) return;
    impala_learn_stats_body(step_stats + (size_t)s * n_sgd * RAMP_IMPALA_STATS_LEN, n_sgd, out + (size_t)s * RAMP_IMPALA_STATS_LEN);
}

// one thread per set: its statistics into its RAMP_PPO_STATS_LEN slice of `out`, where Adam wrote its row count
__global__ void ramp_pop_pg_stats_kernel(const float* row_stats, const int32_t* row_model, const float* adv, int32_t rows, const int32_t* n_rows,
                                         const double* norm_part, double* out, int32_t K) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= K) return;
    pg_stats_body(row_stats + (size_t)s * rows * RS_N, row_model + (size_t)s * rows, adv + (size_t)s * rows, rows, n_rows + s,
                  norm_part + (size_t)s * LRN_GRID, out + (size_t)s * RAMP_PPO_STATS_LEN);
}

// ---- population-based training's exploit: one set's training state onto another ----

struct CopySetsArgs {
    const PopSet* sets;
    const int32_t* pairs;                 // [n_pairs][2]: destination set, source set (equal shapes, checked on the host)
    float* buf[3];                        // [sum n_w] buffers in the population's layout (PopSet::w_off); nullptr: none
    int32_t* step;                        // [K][2] Adam's step counts (both parities), or nullptr
};

// pair `pair`'s source slices onto its destination's, elements chunk blockDim.x + threadIdx.x, grid-strided over n_chunks CTAs
__device__ __forceinline__ void copy_sets_body(const CopySetsArgs& a, int pair, int chunk, int n_chunks) {
    const int d = a.pairs[2 * pair], s = a.pairs[2 * pair + 1];
    const int64_t n = a.sets[d].n_w, od = a.sets[d].w_off, os = a.sets[s].w_off;
    for (int64_t i = (int64_t)chunk * blockDim.x + threadIdx.x; i < n; i += (int64_t)n_chunks * blockDim.x) {
#pragma unroll
        for (int b = 0; b < 3; ++b)
            if (a.buf[b]) a.buf[b][od + i] = a.buf[b][os + i];
    }
    if (a.step && chunk == 0 && threadIdx.x < 2) a.step[2 * d + threadIdx.x] = a.step[2 * s + threadIdx.x];
}

// blockIdx.y = pair, blockIdx.x = chunk: ramp_population_copy_sets and ramp_population_copy_es_sets
__global__ void __launch_bounds__(256) ramp_pop_copy_sets_kernel(const CopySetsArgs a) {
    copy_sets_body(a, blockIdx.y, blockIdx.x, gridDim.x);
}

}  // namespace ramp

// the head-reduce segments of every set for one launch row count
struct PopSegs {
    DeviceArray<Seg> segs; DeviceArray<int32_t> count; DeviceArray<int64_t> first;   // [K][HEAD_SEGS], [K], [K]
    int64_t total = 0;
};

struct ramp_population {
    ramp_policy* p = nullptr;             // the template: job types, act outputs and trajectory (not owned)
    int32_t K = 0;
    std::vector<ramp_policy_config_t> cfgs;   // set s's configuration: the template's environment fields, the rest its own
    std::vector<PopSet> sets;             // host copy of d_sets
    std::vector<uint8_t> has_w;           // set s got weights (ramp_population_set_weights or the template's)
    int64_t nw = 0, n_gpart = 0, n_emb = 0;   // sums over the sets: weights, job-type partials, embeddings
    int32_t rec_stride = 0;               // the largest set's head record
    size_t head_smem = 0;                 // the largest set's read-out staging
    int32_t embed_ctas = 0;               // CTAs of the embedding launches: at most the resident ones
    DeviceArray<PopSet> d_sets;
    DeviceArray<float> d_w, d_emb;        // ragged [K][n_w of the set], [K][n_models][out_node of the set]
    bool emb_valid = false;
    unsigned long long act_calls = 0;
    DeviceArray<unsigned long long> d_seeds, d_keys;
    std::vector<DeviceArray<unsigned char>> gallocs;     // every (set, job type)'s MeanPool states and backward scratch
    LearnerBuffers L;                     // the learner: what ramp_policy keeps for one set, for K (its rec / segs unused: pop_ensure_rows)
    std::map<int32_t, PopSegs> segs;      // every launch row count seen since L.rec was last allocated
    const PopSegs* cur_segs = nullptr;
    DeviceArray<float> d_kl;              // [K][2]: kl_coeff, kl_target
    DeviceArray<GaeArgs> d_gae; DeviceArray<GradArgs> d_grad; DeviceArray<AdamArgs> d_adam;
    DeviceArray<VtraceArgs> d_vtrace;     // IMPALA: every set's V-trace arguments
    DeviceArray<double> d_coef;           // IMPALA: [K][2] vf_loss_coeff, entropy_coeff
    // the copies' (destination, source) pairs: page-locked staging, its device copy, and the end of the last upload from it
    PinnedArray<int32_t> h_pairs;
    DeviceArray<int32_t> d_pairs;
    Event ev_pairs;
};

namespace {

int pop_check_set(const ramp_population* q, int32_t set) {
    if (!q) return set_error(RAMP_ERR_BAD_ARG, "null population");
    if (set < 0 || set >= q->K) return set_error(RAMP_ERR_BAD_ARG, "population: set %d outside [0, %d)", set, q->K);
    return RAMP_OK;
}

// act and learn read every set's weights
int pop_check_weights(const ramp_population* q) {
    for (int s = 0; s < q->K; ++s)
        if (!q->has_w[s]) return set_error(RAMP_ERR_BAD_ARG, "population: set %d has no weights (ramp_population_set_weights)", s);
    return RAMP_OK;
}

// every (set, job type)'s forward states and backward scratch at the set's configuration; the job types' out-edge CSR is the template's
int pop_ensure_gms(ramp_population* q, cudaStream_t st) {
    if (q->L.gmodels_ready) return RAMP_OK;
    ramp_policy* p = q->p;
    const int nm = p->P.c.n_models;
    std::vector<GradModelDev> h((size_t)q->K * nm);
    q->gallocs.clear();
    for (int m = 0; m < nm; ++m) {
        const HostModel& hm = p->models[m];
        if (!hm.set) return set_error(RAMP_ERR_BAD_ARG, "policy: model %d was never registered (ramp_policy_set_model)", m);
        for (int s = 0; s < q->K; ++s) {
            GradModelDev& g = h[(size_t)s * nm + m];
            g = hm.g;
            const int rc = alloc_grad_scratch(q->cfgs[s], hm.d.n_nodes, hm.d.n_edges, q->gallocs, g);
            if (rc != RAMP_OK) return rc;
        }
    }
    return upload_gmodels(q->L, h, st);
}

int pop_launch_embed(ramp_population* q, cudaStream_t st, EmbGradArgs eg, bool forward) {
    ramp_policy* p = q->p;
    PopEmbed pe{};
    pe.K = q->K; pe.n_models = p->P.c.n_models; pe.rec_stride = q->rec_stride;
    if (forward) ramp_pop_embed_grad_kernel<EMB_FORWARD><<<q->embed_ctas, 256, 0, st>>>(q->d_sets.get(), p->d_models.get(), q->L.gmodels.get(), eg, pe);
    else ramp_pop_embed_grad_kernel<EMB_BACKWARD><<<q->embed_ctas, 256, 0, st>>>(q->d_sets.get(), p->d_models.get(), q->L.gmodels.get(), eg, pe);
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

// the embeddings of every set at its current weights (the single policy's act re-embeds the same way when they are stale)
int pop_embed(ramp_population* q, cudaStream_t st) {
    int rc;
    if ((rc = pop_ensure_gms(q, st)) != RAMP_OK) return rc;
    EmbGradArgs eg{};
    eg.emb = q->d_emb.get();
    if ((rc = pop_launch_embed(q, st, eg, true)) != RAMP_OK) return rc;
    q->emb_valid = true;
    return RAMP_OK;
}

// the read-out of `per` rows per set, set s's starting `stride` rows after set s - 1's (0: per)
int pop_launch_head(ramp_population* q, const HeadArgs& a, int32_t per, const unsigned long long* seeds, unsigned long long mix, cudaStream_t st,
                    int32_t stride = 0) {
    ramp_policy* p = q->p;
    const int wpc = 8;
    int gx = (per + wpc - 1) / wpc;
    const int cap = std::max(1, (2 * p->sm_count + q->K - 1) / q->K);      // about the single launch's 2 CTAs per SM in all
    gx = std::max(1, std::min(gx, cap));
    PopHead ph{};
    ph.per = per; ph.stride = stride ? stride : per; ph.seeds = seeds; ph.mix = mix;
    ramp_pop_head_kernel<<<dim3(gx, q->K), wpc * 32, q->head_smem, st>>>(q->d_sets.get(), a, ph);
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

// the learner's buffers, and the per-set arguments of the population's kernels
int pop_ensure_learner(ramp_population* q) {
    if (q->L.ready) return RAMP_OK;
    const size_t K = q->K;
    CUDA_TRY(q->d_kl.alloc(2 * K));
    CUDA_TRY(q->d_gae.alloc(K));
    CUDA_TRY(q->d_grad.alloc(K));
    CUDA_TRY(q->d_adam.alloc(K));
    CUDA_TRY(q->d_vtrace.alloc(K));
    CUDA_TRY(q->d_coef.alloc(2 * K));
    return ensure_learner(q->L, q->nw, q->n_gpart);
}

// ensure_rows for the population: per-row scratch for K launch rows of n rows, set s's at s n rec_stride floats, and every set's
// head segments summing exactly n of its rows, uploaded on `st` the first time n is seen
int pop_ensure_rows(ramp_population* q, int32_t n, cudaStream_t st) {
    LearnerBuffers& L = q->L;
    const size_t K = q->K;
    if (n > L.lcap) {
        const size_t rows = K * n;
        L.lcap = 0;
        q->cur_segs = nullptr;
        q->segs.clear();
        CUDA_TRY(L.rec.alloc(rows * q->rec_stride));
        CUDA_TRY(L.row_stats.alloc(rows * RS_N));
        CUDA_TRY(L.row_model.alloc(rows));
        L.lcap = n;
    }
    auto it = q->segs.find(n);
    if (it == q->segs.end()) {
        std::vector<Seg> h(K * HEAD_SEGS);
        std::vector<int32_t> count(K);
        std::vector<int64_t> first(K);
        PopSegs t;
        for (size_t s = 0; s < K; ++s) {
            Seg* ss = h.data() + s * HEAD_SEGS;
            count[s] = head_segs(q->sets[s].P, L.rec.get() + s * n * q->rec_stride, n, ss);
            first[s] = t.total;
            for (int k = 0; k < count[s]; ++k) {
                const int64_t o = q->sets[s].w_off;
                ss[k].w += o; ss[k].lnw += o; ss[k].lnb += o;
                t.total += seg_size(ss[k]);
            }
        }
        CUDA_TRY(t.segs.alloc(h.size()));
        CUDA_TRY(t.count.alloc(K));
        CUDA_TRY(t.first.alloc(K));
        CUDA_TRY(cudaMemcpyAsync(t.segs.get(), h.data(), sizeof(Seg) * h.size(), cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(t.count.get(), count.data(), sizeof(int32_t) * K, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(t.first.get(), first.data(), sizeof(int64_t) * K, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaStreamSynchronize(st));                              // the vectors are pageable
        it = q->segs.emplace(n, std::move(t)).first;
    }
    q->cur_segs = &it->second;
    return RAMP_OK;
}

// set s's AdamArgs at cfg's settings on its slices of the gradient, moments, step counts, norm partials and weights
template <class Cfg>
AdamArgs pop_adam_args(ramp_population* q, const Cfg& cfg, int s, const int32_t* n_rows, int32_t mb) {
    AdamArgs aa = adam_args(q->p, cfg, n_rows, mb);
    const size_t o = q->sets[s].w_off;
    aa.step = q->L.step.get() + 2 * s; aa.m = q->L.adam_m.get() + o; aa.v = q->L.adam_v.get() + o;
    aa.grad = q->L.grad.get() + o; aa.norm_part = q->L.norm_part.get() + (size_t)s * LRN_GRID; aa.w = q->d_w.get() + o;
    return aa;
}

// every set's configuration, each by its algorithm's own rules; the error names the set
template <class Cfg>
int pop_check_configs(const ramp_population* q, const Cfg* cfgs) {
    if (!q || !cfgs) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    for (int s = 0; s < q->K; ++s)
        if (check_learner_config(&cfgs[s]) != RAMP_OK) return set_error(RAMP_ERR_BAD_ARG, "population: set %d: %s", s, g_last_error.c_str());
    return RAMP_OK;
}

// the opening of the population's learn calls after the configuration checks: learn_begin on the template with set 0's config, a
// trajectory that splits into K groups, the learner's buffers and every (set, job type)'s states on `st`
template <class Cfg>
int pop_learn_begin(ramp_population* q, ramp_engine_t* eng, const Cfg* cfgs, int32_t n_steps, ramp_env_buffers_t* eb, cudaStream_t* st) {
    int rc = learn_begin(q->p, eng, cfgs, n_steps, "population", eb, st);
    if (rc != RAMP_OK || (rc = pop_check_weights(q)) != RAMP_OK) return rc;
    if (eb->n_episodes % q->K)
        return set_error(RAMP_ERR_BAD_ARG, "population: %d episodes do not split into %d groups of equal size", eb->n_episodes, q->K);
    if ((rc = fence_in(q->p, *st)) || (rc = pop_ensure_learner(q)) || (rc = pop_ensure_gms(q, *st))) return rc;
    if ((size_t)q->K > q->d_keys.size()) {                                // the head-gradient kernel reads a key per set (unused unshuffled)
        CUDA_TRY(q->d_keys.alloc(q->K));
        CUDA_TRY(cudaMemsetAsync(q->d_keys.get(), 0, sizeof(unsigned long long) * q->K, *st));
    }
    return RAMP_OK;
}

// head gradient (args: q->d_grad) -> head reduce -> embedding backward -> finish over K launch rows of mb rows each: every set's
// gradient and norm partials.  keys: the [K] shuffle keys (read, and unused, by an unshuffled launch); first_pass: logp_old is written
int pop_launch_grad(ramp_population* q, cudaStream_t st, int32_t mb, int32_t start, const unsigned long long* keys, int first_pass) {
    ramp_policy* p = q->p;
    const int32_t K = q->K;
    const PopSegs* segs = q->cur_segs;
    int64_t rgrid = (segs->total + 255) / 256;
    if (rgrid > 4 * p->sm_count) rgrid = 4 * p->sm_count;
    ramp_pop_head_grad_kernel<<<dim3((mb + LRN_WARPS - 1) / LRN_WARPS, K), LRN_WARPS * 32, 0, st>>>(q->d_sets.get(), q->d_grad.get(), start, keys,
                                                                                                   first_pass);
    ramp_pop_head_reduce_kernel<<<(unsigned)rgrid, 256, 0, st>>>(segs->segs.get(), segs->count.get(), segs->first.get(), K, segs->total,
                                                                 q->d_w.get(), q->L.grad.get());
    CUDA_TRY(cudaGetLastError());
    EmbGradArgs eg{};
    eg.rec = q->L.rec.get(); eg.row_model = q->L.row_model.get(); eg.rows = mb; eg.gpart = q->L.gpart.get();
    int rc = pop_launch_embed(q, st, eg, false);
    if (rc != RAMP_OK) return rc;
    ramp_pop_finish_kernel<<<dim3(LRN_GRID, K), 256, 0, st>>>(q->d_sets.get(), q->L.gpart.get(), p->P.c.n_models, q->L.grad.get(), q->L.norm_part.get());
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

// set s's GAE arguments: its group's b columns of the [T][K b] trajectory, its slice of the train batch; boot: the [K b] bootstrap
// values, or nullptr: no critic (PG)
GaeArgs pop_gae_args(ramp_population* q, int s, int32_t T, int32_t b, double gamma, double lambda, int32_t standardize, const float* boot) {
    ramp_policy* p = q->p;
    const size_t A = p->P.c.n_actions, col = (size_t)s * b, r0 = (size_t)s * T * b;
    GaeArgs ge{};
    ge.T = T; ge.B = b; ge.A = (int32_t)A; ge.n_models = p->P.c.n_models; ge.standardize = standardize; ge.gamma = gamma; ge.lambda = lambda;
    ge.t_obs = p->t_obs.get() + col * 11; ge.t_model = p->t_model.get() + col; ge.t_mask = p->t_mask.get() + col * A;
    ge.t_action = p->t_action.get() + col; ge.t_logp = p->t_logp.get() + col; ge.t_value = boot ? p->t_value.get() + col : nullptr;
    ge.t_reward = p->t_reward.get() + col; ge.t_done = p->t_done.get() + col;
    ge.boot = boot ? boot + col : nullptr; ge.adv64 = q->L.b_adv64.get() + col;
    ge.obs = q->L.b_obs.get() + r0 * 11; ge.model = q->L.b_model.get() + r0; ge.mask = q->L.b_mask.get() + r0 * A; ge.action = q->L.b_action.get() + r0;
    ge.logp = q->L.b_logp.get() + r0; ge.adv = q->L.b_adv.get() + r0; ge.vt = q->L.b_vt.get() + r0; ge.n_rows = q->L.n_rows.get() + s;
    return ge;
}

// set s's head-gradient arguments for launch rows of mb rows: its slices of the per-row scratch and its embeddings
GradArgs pop_grad_args(ramp_population* q, int s, int32_t mb) {
    const size_t q0 = (size_t)s * mb;
    GradArgs ga{};
    ga.mb = mb; ga.graph_static = q->p->d_gstatic.get(); ga.emb = q->d_emb.get() + q->sets[s].emb_off;
    ga.rec = q->L.rec.get() + q0 * q->rec_stride; ga.row_model = q->L.row_model.get() + q0; ga.row_stats = q->L.row_stats.get() + q0 * RS_N;
    return ga;
}

// ramp_population_create_configs' work: the sets' checks, layouts and buffers, no weights yet
int pop_create(ramp_policy* p, int32_t n_sets, const ramp_policy_config_t* cfgs, std::unique_ptr<ramp_population>& out) {
    const ramp_policy_config_t& t = p->P.c;
    std::vector<int64_t> n_w(n_sets);
    int64_t nw = 0;
    size_t smem = 0;
    for (int s = 0; s < n_sets; ++s) {
        const ramp_policy_config_t& c = cfgs[s];
        if (check_config(c) != RAMP_OK) return set_error(RAMP_ERR_BAD_ARG, "population: set %d: %s", s, g_last_error.c_str());
        const char* field = c.in_features_node != t.in_features_node ? "in_features_node" : c.in_features_edge != t.in_features_edge ? "in_features_edge"
                          : c.in_features_graph != t.in_features_graph ? "in_features_graph" : c.n_actions != t.n_actions ? "n_actions"
                          : c.n_models != t.n_models ? "n_models" : nullptr;
        if (field)
            return set_error(RAMP_ERR_BAD_ARG, "population: set %d: %s differs from the template's (the environment and its job types fix it)", s, field);
        const size_t hs = head_smem_floats(c, 8) * sizeof(float);
        if (hs > 200 * 1024) return set_error(RAMP_ERR_CAPACITY, "population: set %d: the read-out needs %zu B of shared memory (max 200 KiB)", s, hs);
        smem = std::max(smem, hs);
        n_w[s] = layout(c, nullptr);
        nw += n_w[s];
    }
    CUDA_TRY(cudaSetDevice(p->device));
    std::unique_ptr<ramp_population> q(new ramp_population());
    q->p = p; q->K = q->L.K = n_sets; q->nw = nw; q->head_smem = smem;
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ramp_pop_embed_grad_kernel<EMB_BACKWARD>, 256, 0));
    q->embed_ctas = std::max(1, std::min(n_sets * t.n_models, std::max(1, per_sm) * p->sm_count));
    CUDA_TRY(reserve_dynamic_smem((const void*)ramp_pop_head_kernel, smem));
    CUDA_TRY(q->d_w.alloc((size_t)nw));
    q->cfgs.assign(cfgs, cfgs + n_sets);
    q->sets.resize(n_sets);
    for (int s = 0; s < n_sets; ++s) {
        PopSet& S = q->sets[s];
        S.P.c = cfgs[s];
        layout(cfgs[s], &S.P);
        S.n_w = n_w[s]; S.w_off = s ? q->sets[s - 1].w_off + n_w[s - 1] : 0; S.P.w = q->d_w.get() + S.w_off;
        S.n_gnn = S.P.gln_w;                                              // the rounds come first in the blob
        S.gpart_off = q->n_gpart; q->n_gpart += (int64_t)t.n_models * S.n_gnn;
        S.emb_off = q->n_emb; q->n_emb += (int64_t)t.n_models * cfgs[s].out_features_node;
        q->rec_stride = std::max(q->rec_stride, head_rec(cfgs[s]).stride);
    }
    q->has_w.assign(n_sets, 0);
    CUDA_TRY(q->d_emb.alloc((size_t)q->n_emb));
    CUDA_TRY(q->d_seeds.alloc(n_sets));
    CUDA_TRY(q->d_sets.alloc(n_sets));
    CUDA_TRY(cudaMemcpy(q->d_sets.get(), q->sets.data(), sizeof(PopSet) * n_sets, cudaMemcpyHostToDevice));
    out = std::move(q);
    return RAMP_OK;
}

// the copies' pairs: sets in [0, K) of equal shape, the source with weights, no set the destination twice, and no set both a source
// and a destination (so the result does not depend on the order the pairs run in).  Errors name the pair.
int pop_check_pairs(const ramp_population* q, int32_t n_pairs, const int32_t* dst, const int32_t* src) {
    if (!q || n_pairs < 0 || (n_pairs > 0 && (!dst || !src))) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n_pairs > 65535) return set_error(RAMP_ERR_BAD_ARG, "population: %d pairs in one copy (max 65535)", n_pairs);
    std::vector<int32_t> as_dst(q->K, -1), as_src(q->K, -1);
    for (int i = 0; i < n_pairs; ++i) {
        const int32_t d = dst[i], s = src[i];
        if (d < 0 || d >= q->K || s < 0 || s >= q->K)
            return set_error(RAMP_ERR_BAD_ARG, "population: pair %d (set %d <- set %d): a set outside [0, %d)", i, d, s, q->K);
        if (memcmp(&q->cfgs[d], &q->cfgs[s], sizeof(ramp_policy_config_t)) != 0)
            return set_error(RAMP_ERR_BAD_ARG, "population: pair %d (set %d <- set %d): the sets differ in shape (ramp_policy_config_t)", i, d, s);
        if (as_dst[d] >= 0)
            return set_error(RAMP_ERR_BAD_ARG, "population: pair %d (set %d <- set %d): set %d is already the destination of pair %d", i, d, s, d,
                             as_dst[d]);
        as_dst[d] = i;
        if (as_src[s] < 0) as_src[s] = i;
        if (!q->has_w[s]) return set_error(RAMP_ERR_BAD_ARG, "population: pair %d (set %d <- set %d): set %d has no weights", i, d, s, s);
    }
    for (int i = 0; i < n_pairs; ++i) {
        const int32_t d = dst[i], s = src[i];
        if (as_src[d] >= 0 || as_dst[s] >= 0)
            return set_error(RAMP_ERR_BAD_ARG, "population: pair %d (set %d <- set %d): set %d is both a source and a destination", i, d, s,
                             as_src[d] >= 0 ? d : s);
    }
    return RAMP_OK;
}

// every pair's source slices of b0..b2 (each [sum n_w] in the population's layout, or nullptr) and, when step is given, its Adam
// step counts onto its destination's: one launch on the default stream, after the template's last fenced call and fenced itself,
// with no host synchronisation.  The pairs were checked (pop_check_pairs).
int pop_copy_sets(ramp_population* q, int32_t n_pairs, const int32_t* dst, const int32_t* src, float* b0, float* b1, float* b2, int32_t* step) {
    if (n_pairs == 0) return RAMP_OK;
    ramp_policy* p = q->p;
    CUDA_TRY(cudaSetDevice(p->device));
    if (!p->ev_done) {                                                    // until now every call kept its own synchronisation
        CUDA_TRY(cudaDeviceSynchronize());
        CUDA_TRY(create(p->ev_done, cudaEventDisableTiming));
    }
    if (!q->ev_pairs) CUDA_TRY(create(q->ev_pairs, cudaEventDisableTiming));
    if (q->h_pairs.size() < 2 * (size_t)q->K) {
        CUDA_TRY(q->h_pairs.alloc(2 * (size_t)q->K));
        CUDA_TRY(q->d_pairs.alloc(2 * (size_t)q->K));
    }
    CUDA_TRY(cudaEventSynchronize(q->ev_pairs.get()));                    // the last copy's upload has read the staging
    int64_t n_max = 0;
    for (int i = 0; i < n_pairs; ++i) {
        q->h_pairs.get()[2 * i] = dst[i];
        q->h_pairs.get()[2 * i + 1] = src[i];
        n_max = std::max(n_max, q->sets[dst[i]].n_w);
    }
    int rc;
    if ((rc = fence_in(p, 0)) != RAMP_OK) return rc;
    CUDA_TRY(cudaMemcpyAsync(q->d_pairs.get(), q->h_pairs.get(), sizeof(int32_t) * 2 * n_pairs, cudaMemcpyHostToDevice, 0));
    CUDA_TRY(cudaEventRecord(q->ev_pairs.get(), 0));
    CopySetsArgs a{};
    a.sets = q->d_sets.get(); a.pairs = q->d_pairs.get(); a.buf[0] = b0; a.buf[1] = b1; a.buf[2] = b2; a.step = step;
    const int chunks = (int)std::max<int64_t>(1, std::min<int64_t>((n_max + 255) / 256, (2 * p->sm_count + n_pairs - 1) / n_pairs));
    ramp_pop_copy_sets_kernel<<<dim3(chunks, n_pairs), 256, 0, 0>>>(a);
    CUDA_TRY(cudaGetLastError());
    return fence_out(p, 0);
}

}  // namespace

extern "C" {

int ramp_population_create_configs(ramp_policy_t* p, int32_t n_sets, const ramp_policy_config_t* cfgs, ramp_population_t** out) {
    if (!p || !cfgs || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n_sets < 1) return set_error(RAMP_ERR_BAD_ARG, "population: %d weight sets", n_sets);
    std::unique_ptr<ramp_population> q;
    const int rc = pop_create(p, n_sets, cfgs, q);
    if (rc != RAMP_OK) return rc;
    *out = q.release();
    return RAMP_OK;
}

int ramp_population_create(ramp_policy_t* p, int32_t n_sets, ramp_population_t** out) {
    if (!p || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n_sets < 1) return set_error(RAMP_ERR_BAD_ARG, "population: %d weight sets", n_sets);
    if (!p->weights_set) return set_error(RAMP_ERR_BAD_ARG, "policy: no weights (ramp_policy_set_weights)");
    const std::vector<ramp_policy_config_t> cfgs(n_sets, p->P.c);
    std::unique_ptr<ramp_population> q;
    const int rc = pop_create(p, n_sets, cfgs.data(), q);
    if (rc != RAMP_OK) return rc;
    CUDA_TRY(cudaDeviceSynchronize());                                    // a running call may still update the template's weights
    for (int s = 0; s < n_sets; ++s)
        CUDA_TRY(cudaMemcpy(q->d_w.get() + q->sets[s].w_off, p->d_w.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToDevice));
    q->has_w.assign(n_sets, 1);
    *out = q.release();
    return RAMP_OK;
}

void ramp_population_destroy(ramp_population_t* q) {
    if (!q) return;
    cudaSetDevice(q->p->device);
    delete q;
}

int ramp_population_set_weights(ramp_population_t* q, int32_t set, const float* weights, int64_t n) {
    int rc = pop_check_set(q, set);
    if (rc != RAMP_OK) return rc;
    if (!weights) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    const PopSet& S = q->sets[set];
    if (n != S.n_w)
        return set_error(RAMP_ERR_BAD_ARG, "population: %lld weights given for set %d, its configuration has %lld", (long long)n, set, (long long)S.n_w);
    CUDA_TRY(cudaSetDevice(q->p->device));
    CUDA_TRY(cudaDeviceSynchronize());                                    // a running rollout may still read the old set
    CUDA_TRY(cudaMemcpy(q->d_w.get() + S.w_off, weights, sizeof(float) * n, cudaMemcpyHostToDevice));
    q->has_w[set] = 1;
    q->emb_valid = false;
    return RAMP_OK;
}

int ramp_population_get_weights(ramp_population_t* q, int32_t set, float* out) {
    int rc = pop_check_set(q, set);
    if (rc != RAMP_OK) return rc;
    if (!out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    const PopSet& S = q->sets[set];
    CUDA_TRY(cudaSetDevice(q->p->device));
    CUDA_TRY(cudaDeviceSynchronize());                                    // a learn call may still be updating them
    CUDA_TRY(cudaMemcpy(out, q->d_w.get() + S.w_off, sizeof(float) * S.n_w, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_population_act(ramp_population_t* q, ramp_engine_t* eng, int32_t sample, const uint64_t* seeds) {
    if (!q || !eng || (sample && !seeds)) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    ramp_policy* p = q->p;
    ramp_env_buffers_t eb{};
    int rc = ramp_env_buffers(eng, &eb);
    if (rc != RAMP_OK) return rc;
    const ramp_policy_config_t& c = p->P.c;
    if (ramp_internal_device(eng) != p->device) return set_error(RAMP_ERR_BAD_ARG, "policy and engine live on different devices");
    if (eb.n_actions != c.n_actions) return set_error(RAMP_ERR_BAD_ARG, "policy has %d actions, the environment %d", c.n_actions, eb.n_actions);
    if (c.in_features_graph != 17) return set_error(RAMP_ERR_BAD_ARG, "the environment emits 17 graph features, the policy expects %d", c.in_features_graph);
    if (eb.n_models > c.n_models) return set_error(RAMP_ERR_BAD_ARG, "the environment has %d job types, the policy %d", eb.n_models, c.n_models);
    if (eb.n_episodes % q->K)
        return set_error(RAMP_ERR_BAD_ARG, "population: %d episodes do not split into %d groups of equal size", eb.n_episodes, q->K);
    if ((rc = pop_check_weights(q)) != RAMP_OK) return rc;
    CUDA_TRY(cudaSetDevice(p->device));
    cudaStream_t st = ramp_internal_stream(eng);
    int launches = 1;
    if ((rc = fence_in(p, st)) != RAMP_OK) return rc;
    if (!q->emb_valid) { if ((rc = pop_embed(q, st)) != RAMP_OK) return rc; ++launches; }
    if ((rc = ensure_outputs(p, eb.n_episodes)) != RAMP_OK) return rc;
    if (sample) CUDA_TRY(cudaMemcpyAsync(q->d_seeds.get(), seeds, sizeof(uint64_t) * q->K, cudaMemcpyHostToDevice, st));
    HeadArgs a{};
    a.obs_dyn = eb.obs_dynamic; a.graph_static = p->d_gstatic.get(); a.model = eb.queued_model; a.done = eb.done;
    a.mask = eb.action_mask; a.emb = q->d_emb.get(); a.logits = p->d_logits.get(); a.value = p->d_value.get(); a.logp = p->d_logp.get(); a.actions = eb.actions;
    a.sample = sample;
    if ((rc = pop_launch_head(q, a, eb.n_episodes / q->K, q->d_seeds.get(), 0x9E3779B97F4A7C15ull * (++q->act_calls), st)) != RAMP_OK ||
        (rc = fence_out(p, st)) != RAMP_OK)
        return rc;
    p->act_n = eb.n_episodes;                                             // ramp_policy_read and the trajectory take act's outputs
    ramp_internal_count_launches(eng, launches);
    return RAMP_OK;
}

int ramp_population_learn(ramp_population_t* q, ramp_engine_t* eng, int32_t n_steps, const ramp_ppo_config_t* cfgs, double* stats_out) {
    if (!q || !cfgs) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    ramp_policy* p = q->p;
    const int32_t K = q->K;
    for (int s = 0; s < K; ++s) {
        int rc = check_learner_config(&cfgs[s]);
        if (rc != RAMP_OK) return rc;
        if (cfgs[s].sgd_minibatch_size != cfgs[0].sgd_minibatch_size)
            return set_error(RAMP_ERR_BAD_ARG, "population: sgd_minibatch_size of set %d (%d) differs from set 0's (%d)", s,
                             cfgs[s].sgd_minibatch_size, cfgs[0].sgd_minibatch_size);
        if (cfgs[s].num_sgd_iter != cfgs[0].num_sgd_iter)
            return set_error(RAMP_ERR_BAD_ARG, "population: num_sgd_iter of set %d (%d) differs from set 0's (%d)", s,
                             cfgs[s].num_sgd_iter, cfgs[0].num_sgd_iter);
    }
    ramp_env_buffers_t eb{};
    cudaStream_t st;
    int rc = pop_learn_begin(q, eng, cfgs, n_steps, &eb, &st);
    if (rc != RAMP_OK) return rc;
    const ramp_policy_config_t& c = p->P.c;
    const int32_t B = eb.n_episodes, b = B / K, rows = n_steps * b, mb = cfgs[0].sgd_minibatch_size, n_mb = (rows + mb - 1) / mb;
    const int32_t n_pass = cfgs[0].num_sgd_iter, A = c.n_actions;
    const size_t R = rows;
    if ((rc = pop_ensure_rows(q, mb, st)) || (rc = ensure_batch(q->L, c, rows)) || (rc = ensure_ppo(q->L, B, n_mb))) return rc;
    if (!q->emb_valid && (rc = pop_embed(q, st)) != RAMP_OK) return rc;
    if ((size_t)K * std::max(n_pass, 1) > q->d_keys.size()) CUDA_TRY(q->d_keys.alloc((size_t)K * std::max(n_pass, 1)));
    // every group's arguments: set s's slices of the trajectory's columns, the train batch, the scratch and the learner state
    std::vector<GaeArgs> gae(K);
    std::vector<GradArgs> grad(K);
    std::vector<AdamArgs> adam(K);
    std::vector<float> kl(2 * K);
    std::vector<unsigned long long> keys((size_t)K * std::max(n_pass, 1));
    const float* boot = p->t_value.get() + (size_t)n_steps * B;
    if (n_steps == p->traj_n) boot = q->L.boot.get();
    for (int s = 0; s < K; ++s) {
        const ramp_ppo_config_t& cfg = cfgs[s];
        const size_t r0 = (size_t)s * R;
        gae[s] = pop_gae_args(q, s, n_steps, b, cfg.gamma, cfg.lambda, cfg.standardize_advantages, boot);
        GradArgs& ga = grad[s];
        ga = pop_grad_args(q, s, mb);
        ga.n_rows = q->L.n_rows.get() + s; ga.shuffle = 1; ga.obs_dyn = q->L.b_obs.get() + r0 * 11; ga.model = q->L.b_model.get() + r0;
        ga.mask = q->L.b_mask.get() + r0 * A; ga.action = q->L.b_action.get() + r0; ga.old_logits = q->L.b_old.get() + r0 * A;
        ga.adv = q->L.b_adv.get() + r0; ga.vt = q->L.b_vt.get() + r0; ga.logp_old = q->L.b_logp_old.get() + r0;
        ppo_terms(ga, cfg);
        AdamArgs& aa = adam[s];
        aa = pop_adam_args(q, cfg, s, q->L.n_rows.get() + s, mb);
        aa.row_stats = ga.row_stats; aa.vf_coeff = ga.vf_coeff; aa.ent_coeff = ga.ent_coeff; aa.kl_coeff = ga.kl_coeff;
        aa.stats = q->L.mb_stats.get() + (size_t)s * n_mb * RAMP_PPO_STATS_LEN;
        kl[2 * s] = (float)cfg.kl_coeff; kl[2 * s + 1] = (float)cfg.kl_target;
        for (int pass = 0; pass < n_pass; ++pass) keys[(size_t)pass * K + s] = mix64(cfg.seed ^ mix64((uint64_t)pass + 1));
    }
    CUDA_TRY(cudaMemcpyAsync(q->d_gae.get(), gae.data(), sizeof(GaeArgs) * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(q->d_grad.get(), grad.data(), sizeof(GradArgs) * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(q->d_adam.get(), adam.data(), sizeof(AdamArgs) * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(q->d_kl.get(), kl.data(), sizeof(float) * 2 * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(q->d_keys.get(), keys.data(), sizeof(unsigned long long) * keys.size(), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));                                  // the vectors are pageable
    int launches = 2;                                                     // GAE, old logits
    // 1. the value of the state after the last step, as ramp_policy_learn takes it
    if (n_steps == p->traj_n) {
        HeadArgs hb{};
        hb.obs_dyn = eb.obs_dynamic; hb.graph_static = p->d_gstatic.get(); hb.model = eb.queued_model; hb.done = eb.done;
        hb.mask = eb.action_mask; hb.emb = q->d_emb.get(); hb.value = q->L.boot.get(); hb.actions = q->L.boot_act.get();
        if ((rc = pop_launch_head(q, hb, b, nullptr, 0, st)) != RAMP_OK) return rc;
        ++launches;
    }
    // 2. GAE, one CTA per group
    ramp_pop_gae_kernel<<<K, 1024, 0, st>>>(q->d_gae.get(), B);
    CUDA_TRY(cudaGetLastError());
    // 3. the collection weights' logits of every row
    HeadArgs ho{};
    ho.obs_dyn = q->L.b_obs.get(); ho.graph_static = p->d_gstatic.get(); ho.model = q->L.b_model.get(); ho.mask = q->L.b_mask.get();
    ho.emb = q->d_emb.get(); ho.logits = q->L.b_old.get(); ho.value = q->L.b_value.get(); ho.logp = q->L.b_lpx.get(); ho.actions = q->L.b_actx.get();
    if ((rc = pop_launch_head(q, ho, rows, nullptr, 0, st)) != RAMP_OK) return rc;
    // 4. minibatch j of every group in the same launches
    for (int pass = 0; pass < n_pass; ++pass) {
        for (int j = 0; j < n_mb; ++j) {
            const int32_t start = j * mb;
            EmbGradArgs ef{};
            ef.n_rows = q->L.n_rows.get(); ef.start = start; ef.emb = pass || j ? q->d_emb.get() : nullptr;
            if ((rc = pop_launch_embed(q, st, ef, true)) != RAMP_OK ||
                (rc = pop_launch_grad(q, st, mb, start, q->d_keys.get() + (size_t)pass * K, pass == 0)) != RAMP_OK)
                return rc;
            ramp_pop_adam_kernel<<<dim3(LRN_GRID, K), 256, 0, st>>>(q->d_sets.get(), q->d_adam.get(), start, j, q->L.parity);
            q->L.parity ^= 1;
            CUDA_TRY(cudaGetLastError());
            launches += 6;
        }
    }
    if (n_pass > 0) q->emb_valid = false;
    // 5. every set's last-pass statistics and adapted KL coefficient: the call's one read-back
    ramp_pop_learn_stats_kernel<<<(K + 127) / 128, 128, 0, st>>>(q->L.mb_stats.get(), n_mb, n_pass > 0 ? n_mb : 0, q->d_kl.get(),
                                                                q->L.n_rows.get(), q->L.stats.get(), K);
    CUDA_TRY(cudaGetLastError());
    ramp_internal_count_launches(eng, launches + 1);
    if (stats_out) CUDA_TRY(cudaMemcpyAsync(stats_out, q->L.stats.get(), sizeof(double) * K * RAMP_PPO_STATS_LEN, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return fence_out(p, st);
}

int ramp_population_learn_impala(ramp_population_t* q, ramp_engine_t* eng, int32_t n_steps, const ramp_impala_config_t* cfgs, double* stats_out) {
    int rc = pop_check_configs(q, cfgs);
    if (rc != RAMP_OK) return rc;
    ramp_policy* p = q->p;
    const int32_t K = q->K;
    for (int s = 1; s < K; ++s) {
        if (cfgs[s].rollout_fragment_length != cfgs[0].rollout_fragment_length)
            return set_error(RAMP_ERR_BAD_ARG, "population: rollout_fragment_length of set %d (%d) differs from set 0's (%d)", s,
                             cfgs[s].rollout_fragment_length, cfgs[0].rollout_fragment_length);
        if (cfgs[s].train_batch_size != cfgs[0].train_batch_size)
            return set_error(RAMP_ERR_BAD_ARG, "population: train_batch_size of set %d (%d) differs from set 0's (%d)", s,
                             cfgs[s].train_batch_size, cfgs[0].train_batch_size);
    }
    ramp_env_buffers_t eb{};
    cudaStream_t st;
    if ((rc = pop_learn_begin(q, eng, cfgs, n_steps, &eb, &st)) != RAMP_OK) return rc;
    const int32_t L = cfgs[0].rollout_fragment_length ? cfgs[0].rollout_fragment_length : n_steps;
    if (n_steps % L) return set_error(RAMP_ERR_BAD_ARG, "impala: rollout_fragment_length %d does not divide %d steps", L, n_steps);
    if (cfgs[0].train_batch_size < L)
        return set_error(RAMP_ERR_BAD_ARG, "impala: train_batch_size %d is below rollout_fragment_length %d", cfgs[0].train_batch_size, L);
    const ramp_policy_config_t& c = p->P.c;
    const int32_t b = eb.n_episodes / K, n_frag = (n_steps / L) * b, R = n_steps * b, A = c.n_actions;
    const int32_t F = std::min(cfgs[0].train_batch_size / L, n_frag), mb = F * L, n_sgd = (n_frag + F - 1) / F;
    if ((rc = pop_ensure_rows(q, mb, st)) || (rc = ensure_impala(q->L, c, R, n_sgd))) return rc;
    if (!q->emb_valid && (rc = pop_embed(q, st)) != RAMP_OK) return rc;
    LearnerBuffers& Lb = q->L;
    // every set's arguments: its slices of the fragment rows, the per-row scratch and the learner state
    std::vector<VtraceArgs> vt(K);
    std::vector<GradArgs> grad(K);
    std::vector<AdamArgs> adam(K);
    std::vector<double> coef(2 * K);
    for (int s = 0; s < K; ++s) {
        const ramp_impala_config_t& cfg = cfgs[s];
        const size_t r0 = (size_t)s * R;
        VtraceArgs& v = vt[s];
        v.L = L; v.A = A; v.n_models = c.n_models;
        v.gamma = cfg.gamma; v.clip_rho = cfg.vtrace_clip_rho_threshold; v.clip_pg_rho = cfg.vtrace_clip_pg_rho_threshold;
        v.logits = Lb.i_tlogits.get() + r0 * A; v.value = Lb.i_tvalue.get() + r0;
        v.model = Lb.i_model.get() + r0; v.action = Lb.i_action.get() + r0; v.blogp = Lb.i_blogp.get() + r0; v.reward = Lb.i_reward.get() + r0;
        v.done = Lb.i_done.get() + r0; v.tlogp = Lb.i_tlogp.get() + r0; v.log_rho = Lb.i_log_rho.get() + r0; v.vs = Lb.i_vs.get() + r0;
        v.pg_adv = Lb.i_pg.get() + r0; v.lmodel = Lb.i_lmodel.get() + r0;
        GradArgs& ga = grad[s];
        ga = pop_grad_args(q, s, mb);
        ga.n_rows = Lb.i_n_rows.get() + s; ga.impala = 1; ga.obs_dyn = Lb.i_obs.get() + r0 * 11; ga.model = Lb.i_lmodel.get() + r0;
        ga.mask = Lb.i_mask.get() + r0 * A; ga.action = Lb.i_action.get() + r0; ga.adv = Lb.i_pg.get() + r0; ga.vt = Lb.i_vs.get() + r0;
        ga.vf_coeff = (float)cfg.vf_loss_coeff; ga.ent_coeff = (float)cfg.entropy_coeff;
        adam[s] = pop_adam_args(q, cfg, s, Lb.i_n_rows.get() + s, mb);
        adam[s].stats = Lb.i_stats.get() + (size_t)s * RAMP_IMPALA_STATS_LEN;
        coef[2 * s] = cfg.vf_loss_coeff; coef[2 * s + 1] = cfg.entropy_coeff;
    }
    CUDA_TRY(cudaMemcpyAsync(q->d_vtrace.get(), vt.data(), sizeof(VtraceArgs) * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(q->d_grad.get(), grad.data(), sizeof(GradArgs) * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(q->d_adam.get(), adam.data(), sizeof(AdamArgs) * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(q->d_coef.get(), coef.data(), sizeof(double) * 2 * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));                                  // the vectors are pageable
    // 1. every group's fragment rows, fragment-major
    ImpalaBatchArgs ba{};
    ba.T = n_steps; ba.B = b; ba.A = A; ba.L = L; ba.n_models = c.n_models;
    ba.t_obs = p->t_obs.get(); ba.t_model = p->t_model.get(); ba.t_mask = p->t_mask.get(); ba.t_action = p->t_action.get();
    ba.t_logp = p->t_logp.get(); ba.t_reward = p->t_reward.get(); ba.t_done = p->t_done.get();
    ba.obs = Lb.i_obs.get(); ba.model = Lb.i_model.get(); ba.mask = Lb.i_mask.get(); ba.action = Lb.i_action.get();
    ba.blogp = Lb.i_blogp.get(); ba.reward = Lb.i_reward.get(); ba.done = Lb.i_done.get(); ba.n_rows = Lb.i_n_rows.get();
    ramp_pop_impala_batch_kernel<<<(unsigned)(((int64_t)K * R + 255) / 256), 256, 0, st>>>(ba, K);
    CUDA_TRY(cudaGetLastError());
    // 2. SGD step k of every set in the same launches
    for (int k = 0; k < n_sgd; ++k) {
        const int32_t start = k * mb, nf = std::min(F, n_frag - k * F);
        // the rounds at the current weights, kept for the backward; from the second step on also the embeddings
        EmbGradArgs ef{};
        ef.n_rows = Lb.i_n_rows.get(); ef.start = start; ef.emb = k ? q->d_emb.get() : nullptr;
        if ((rc = pop_launch_embed(q, st, ef, true)) != RAMP_OK) return rc;
        // the read-out of the step's fragment rows at the current weights: rows [s R + start, s R + start + nf L) of set s
        HeadArgs h{};
        h.obs_dyn = Lb.i_obs.get() + (size_t)start * 11; h.graph_static = p->d_gstatic.get(); h.model = Lb.i_model.get() + start;
        h.mask = Lb.i_mask.get() + (size_t)start * A; h.emb = q->d_emb.get(); h.logits = Lb.i_tlogits.get() + (size_t)start * A;
        h.value = Lb.i_tvalue.get() + start; h.actions = Lb.i_actx.get() + start;
        if ((rc = pop_launch_head(q, h, nf * L, nullptr, 0, st, R)) != RAMP_OK) return rc;
        ramp_pop_vtrace_kernel<<<(unsigned)((K * nf + 7) / 8), 256, 0, st>>>(q->d_vtrace.get(), K, nf, start);
        CUDA_TRY(cudaGetLastError());
        if ((rc = pop_launch_grad(q, st, mb, start, q->d_keys.get(), 1)) != RAMP_OK) return rc;
        ramp_pop_adam_kernel<<<dim3(LRN_GRID, K), 256, 0, st>>>(q->d_sets.get(), q->d_adam.get(), start, 0, Lb.parity);
        Lb.parity ^= 1;
        ramp_pop_impala_step_stats_kernel<<<(K + 127) / 128, 128, 0, st>>>(Lb.row_stats.get(), Lb.row_model.get(), mb, start, Lb.i_log_rho.get(), R,
                                                                          q->d_coef.get(), Lb.norm_part.get(), Lb.i_step_stats.get(), n_sgd, k, K);
        CUDA_TRY(cudaGetLastError());
    }
    q->emb_valid = false;
    Lb.i_rows = R;
    // 3. every set's means over its steps: the call's one read-back
    ramp_pop_impala_learn_stats_kernel<<<(K + 127) / 128, 128, 0, st>>>(Lb.i_step_stats.get(), n_sgd, Lb.i_stats.get(), K);
    CUDA_TRY(cudaGetLastError());
    ramp_internal_count_launches(eng, 2 + 9 * n_sgd);
    if (stats_out) CUDA_TRY(cudaMemcpyAsync(stats_out, Lb.i_stats.get(), sizeof(double) * K * RAMP_IMPALA_STATS_LEN, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return fence_out(p, st);
}

int ramp_population_learn_pg(ramp_population_t* q, ramp_engine_t* eng, int32_t n_steps, const ramp_pg_config_t* cfgs, double* stats_out) {
    int rc = pop_check_configs(q, cfgs);
    if (rc != RAMP_OK) return rc;
    ramp_policy* p = q->p;
    const int32_t K = q->K;
    ramp_env_buffers_t eb{};
    cudaStream_t st;
    if ((rc = pop_learn_begin(q, eng, cfgs, n_steps, &eb, &st)) != RAMP_OK) return rc;
    const ramp_policy_config_t& c = p->P.c;
    const int32_t b = eb.n_episodes / K, rows = n_steps * b, A = c.n_actions;
    if ((rc = pop_ensure_rows(q, rows, st)) || (rc = ensure_batch(q->L, c, rows))) return rc;
    if (!q->emb_valid && (rc = pop_embed(q, st)) != RAMP_OK) return rc;
    LearnerBuffers& Lb = q->L;
    std::vector<GaeArgs> gae(K);
    std::vector<GradArgs> grad(K);
    std::vector<AdamArgs> adam(K);
    for (int s = 0; s < K; ++s) {
        const ramp_pg_config_t& cfg = cfgs[s];
        const size_t r0 = (size_t)s * rows;
        gae[s] = pop_gae_args(q, s, n_steps, b, cfg.gamma, 1.0, 0, nullptr);
        GradArgs& ga = grad[s];
        ga = pop_grad_args(q, s, rows);
        ga.n_rows = Lb.n_rows.get() + s; ga.pg = 1; ga.obs_dyn = Lb.b_obs.get() + r0 * 11; ga.model = Lb.b_model.get() + r0;
        ga.mask = Lb.b_mask.get() + r0 * A; ga.action = Lb.b_action.get() + r0; ga.adv = Lb.b_adv.get() + r0; ga.logp_old = Lb.b_logp_old.get() + r0;
        adam[s] = pop_adam_args(q, cfg, s, Lb.n_rows.get() + s, rows);
        adam[s].stats = Lb.stats.get() + (size_t)s * RAMP_PPO_STATS_LEN;
    }
    CUDA_TRY(cudaMemcpyAsync(q->d_gae.get(), gae.data(), sizeof(GaeArgs) * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(q->d_grad.get(), grad.data(), sizeof(GradArgs) * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(q->d_adam.get(), adam.data(), sizeof(AdamArgs) * K, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));                                  // the vectors are pageable
    // 1. every group's discounted returns, its live rows t-major into its slice of the train batch
    ramp_pop_gae_kernel<<<K, 1024, 0, st>>>(q->d_gae.get(), eb.n_episodes);
    CUDA_TRY(cudaGetLastError());
    // 2. the loss's gradient over each group's whole batch at the collection weights
    EmbGradArgs ef{};
    ef.n_rows = Lb.n_rows.get();
    if ((rc = pop_launch_embed(q, st, ef, true)) != RAMP_OK || (rc = pop_launch_grad(q, st, rows, 0, q->d_keys.get(), 1)) != RAMP_OK) return rc;
    // 3. one Adam step per set; a set with no row makes none and keeps its step count
    ramp_pop_adam_kernel<<<dim3(LRN_GRID, K), 256, 0, st>>>(q->d_sets.get(), q->d_adam.get(), 0, 0, Lb.parity);
    Lb.parity ^= 1;
    // 4. the statistics: the call's one read-back
    ramp_pop_pg_stats_kernel<<<(K + 127) / 128, 128, 0, st>>>(Lb.row_stats.get(), Lb.row_model.get(), Lb.b_adv.get(), rows, Lb.n_rows.get(),
                                                              Lb.norm_part.get(), Lb.stats.get(), K);
    CUDA_TRY(cudaGetLastError());
    q->emb_valid = false;
    ramp_internal_count_launches(eng, 8);
    if (stats_out)
        CUDA_TRY(cudaMemcpy2DAsync(stats_out, sizeof(double) * RAMP_PG_STATS_LEN, Lb.stats.get(), sizeof(double) * RAMP_PPO_STATS_LEN,
                                   sizeof(double) * RAMP_PG_STATS_LEN, K, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return fence_out(p, st);
}

int ramp_population_vtrace_read(ramp_population_t* q, int32_t set, int32_t* n_out, float* target_logp_out, float* log_rho_out, float* vs_out,
                                float* pg_adv_out) {
    int rc = pop_check_set(q, set);
    if (rc != RAMP_OK) return rc;
    if (!n_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (q->L.i_rows < 1) return set_error(RAMP_ERR_BAD_ARG, "population: no V-trace yet (ramp_population_learn_impala)");
    CUDA_TRY(cudaSetDevice(q->p->device));
    CUDA_TRY(cudaDeviceSynchronize());
    const size_t n = q->L.i_rows, o = (size_t)set * n;
    *n_out = q->L.i_rows;
    if (target_logp_out) CUDA_TRY(cudaMemcpy(target_logp_out, q->L.i_tlogp.get() + o, 4 * n, cudaMemcpyDeviceToHost));
    if (log_rho_out) CUDA_TRY(cudaMemcpy(log_rho_out, q->L.i_log_rho.get() + o, 4 * n, cudaMemcpyDeviceToHost));
    if (vs_out) CUDA_TRY(cudaMemcpy(vs_out, q->L.i_vs.get() + o, 4 * n, cudaMemcpyDeviceToHost));
    if (pg_adv_out) CUDA_TRY(cudaMemcpy(pg_adv_out, q->L.i_pg.get() + o, 4 * n, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_population_learner_state(ramp_population_t* q, int32_t set, float* exp_avg_out, float* exp_avg_sq_out, int32_t* step_out) {
    int rc = pop_check_set(q, set);
    if (rc != RAMP_OK) return rc;
    CUDA_TRY(cudaSetDevice(q->p->device));
    const size_t n = q->sets[set].n_w, o = q->sets[set].w_off;
    if (!q->L.ready) {
        if (exp_avg_out) memset(exp_avg_out, 0, sizeof(float) * n);
        if (exp_avg_sq_out) memset(exp_avg_sq_out, 0, sizeof(float) * n);
        if (step_out) *step_out = 0;
        return RAMP_OK;
    }
    CUDA_TRY(cudaDeviceSynchronize());                                    // a learn call may still be updating them
    if (exp_avg_out) CUDA_TRY(cudaMemcpy(exp_avg_out, q->L.adam_m.get() + o, sizeof(float) * n, cudaMemcpyDeviceToHost));
    if (exp_avg_sq_out) CUDA_TRY(cudaMemcpy(exp_avg_sq_out, q->L.adam_v.get() + o, sizeof(float) * n, cudaMemcpyDeviceToHost));
    if (step_out) CUDA_TRY(cudaMemcpy(step_out, q->L.step.get() + 2 * set + q->L.parity, sizeof(int32_t), cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_population_set_learner_state(ramp_population_t* q, int32_t set, const float* exp_avg, const float* exp_avg_sq, int64_t n, int32_t step) {
    int rc = pop_check_set(q, set);
    if (rc != RAMP_OK) return rc;
    if (!exp_avg || !exp_avg_sq) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    const PopSet& S = q->sets[set];
    if (n != S.n_w)
        return set_error(RAMP_ERR_BAD_ARG, "population: a learner state of %lld weights given for set %d, its configuration has %lld", (long long)n, set,
                         (long long)S.n_w);
    if (step < 0) return set_error(RAMP_ERR_BAD_ARG, "population: set %d: Adam step count %d < 0", set, step);
    CUDA_TRY(cudaSetDevice(q->p->device));
    if ((rc = pop_ensure_learner(q)) != RAMP_OK) return rc;
    CUDA_TRY(cudaDeviceSynchronize());                                    // a learn call may still be updating them
    CUDA_TRY(cudaMemcpy(q->L.adam_m.get() + S.w_off, exp_avg, sizeof(float) * n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(q->L.adam_v.get() + S.w_off, exp_avg_sq, sizeof(float) * n, cudaMemcpyHostToDevice));
    const int32_t steps[2] = {step, step};
    CUDA_TRY(cudaMemcpy(q->L.step.get() + 2 * set, steps, sizeof(steps), cudaMemcpyHostToDevice));
    return RAMP_OK;
}

int ramp_population_copy_sets(ramp_population_t* q, int32_t n_pairs, const int32_t* dst, const int32_t* src) {
    int rc = pop_check_pairs(q, n_pairs, dst, src);
    if (rc != RAMP_OK) return rc;
    LearnerBuffers& L = q->L;                                             // before the first learn call every Adam state is zero
    if ((rc = pop_copy_sets(q, n_pairs, dst, src, q->d_w.get(), L.ready ? L.adam_m.get() : nullptr, L.ready ? L.adam_v.get() : nullptr,
                            L.ready ? L.step.get() : nullptr)) != RAMP_OK)
        return rc;
    for (int i = 0; i < n_pairs; ++i) q->has_w[dst[i]] = 1;
    if (n_pairs > 0) q->emb_valid = false;
    return RAMP_OK;
}

int ramp_population_get_act_count(ramp_population_t* q, uint64_t* out) {
    if (!q || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    *out = q->act_calls;
    return RAMP_OK;
}

int ramp_population_set_act_count(ramp_population_t* q, uint64_t n) {
    if (!q) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    q->act_calls = n;
    return RAMP_OK;
}

int ramp_population_embed_ctas(ramp_population_t* q, int32_t* ctas_out) {
    if (!q || !ctas_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    *ctas_out = q->embed_ctas;
    return RAMP_OK;
}

}  // extern "C"
