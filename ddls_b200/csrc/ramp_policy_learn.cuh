// ramp_policy_learn.cuh -- the GNN policy's gradient and RLlib's PPO learner step on the device (include/ramp_b200.h:
// ramp_policy_backward, ramp_ppo_loss_grad, ramp_policy_learn), RLlib's IMPALA learner step (ramp_impala_loss_grad,
// ramp_policy_learn_impala) and RLlib's PG learner step (ramp_pg_loss_grad, ramp_policy_learn_pg).  Included by ramp_policy.cu after the forward kernels: the forwards recomputed here repeat theirs
// operation for operation, so a recomputed logit is the one ramp_policy_act produced, bit for bit.
//
//   ramp_policy_head_grad_kernel    one warp per row: the read-out forward, the upstream gradient (given, RLlib's PPO loss,
//                                   IMPALA's VTraceLoss or PG's loss), and
//                                   its backward through the logits / value layers, both hidden layers and the graph module; a
//                                   per-row record of what the weight gradients need
//   ramp_policy_head_reduce_kernel  one thread per read-out / graph-module weight: its gradient summed over the rows in row order
//   ramp_gnn_embed_grad_kernel      one CTA per job type, two launches: before the head gradient the MeanPool rounds, every
//                                   round's states kept (and the embeddings the minibatch reads); after it, d emb from the rows in
//                                   row order, backward round by round; a source node's message gradients are gathered through an
//                                   out-edge CSR; the job type's weight gradients summed over its items in order
//   ramp_grad_finish_kernel         the job types' gradients summed in model order; per-CTA partial squared norms
//   ramp_adam_kernel                clip_grad_norm_ + torch.optim.Adam; the minibatch's loss statistics
//   ramp_ppo_gae_kernel             GAE per episode, t-major compaction of the live rows, advantage standardisation; without
//                                   values (PG) the discounted returns
//   ramp_ppo_learn_stats_kernel     the last pass's mean statistics and RLlib's KL-coefficient update
//   ramp_impala_batch_kernel        the trajectory cut into fragments of L rows, fragment-major
//   ramp_vtrace_kernel              one warp per fragment: target log-probabilities (the head kernel's log-softmax), V-trace in f64
//   ramp_impala_*_stats_kernel      one SGD step's IMPALA statistics; the call's means over its steps
//   ramp_pg_stats_kernel            PG's statistics
//
// Every weight gradient is a sum in a fixed order with an f64 accumulator and no atomics: one call on one batch gives the same bits.
#pragma once

namespace ramp {

constexpr int LRN_WARPS = 8;             // rows per CTA of the head-gradient kernel
constexpr int LRN_GRID = 264;            // CTAs of the finish / Adam kernels: the norm's partials always sum in one order
enum { RS_PI, RS_VF, RS_ENT, RS_KL, RS_CLIP, RS_N };   // per-row PPO terms

// offsets (floats) of one row's record of the head-gradient kernel
struct HeadRec { int32_t xg, dyg, dpg, fb, de, h, hv, dh, dhv, dl, dv, stride; };

__host__ __device__ inline HeadRec head_rec(const ramp_policy_config_t& c) {
    const int gin = c.in_features_graph + c.n_actions, og = c.out_features_graph, on = c.out_features_node, fin = on + og;
    const int H = c.fcnet_hidden, A = c.n_actions;
    HeadRec r{};
    int o = 0;
    r.xg = o; o += gin;                  // LayerNorm-normalised [graph features | mask]
    r.dyg = o; o += gin;                 // d graph-module LayerNorm output
    r.dpg = o; o += og;                  // d graph-module Linear output
    r.fb = o; o += fin;                  // read-out input
    r.de = o; o += on;                   // d emb[model]
    r.h = o; o += H; r.hv = o; o += H;   // hidden activations (policy, value)
    r.dh = o; o += H; r.dhv = o; o += H; // d hidden pre-activations
    r.dl = o; o += A; r.dv = o; o += 1;  // d logits, d value
    r.stride = o;
    return r;
}

// one weight tensor's gradient as a sum over the items of a record array, item by item (f64):
//   OUTER     g[o][k] = sum a[o] b[k]        OUTER_LN  the same with b[k] -> b[k] lnw[k] + lnb[k] (LayerNorm output from x-hat)
//   SUM       g[o]    = sum a[o]             DOT       g[k]    = sum a[k] b[k]
enum { SEG_OUTER, SEG_OUTER_LN, SEG_SUM, SEG_DOT };
struct Seg {
    const float* rec;
    int32_t stride, n, kind, O, K, a, b;
    int64_t w, lnw, lnb;                 // blob offsets: the tensor, and the LayerNorm affine of OUTER_LN
};

__host__ __device__ inline int64_t seg_size(const Seg& s) {
    return s.kind == SEG_SUM ? s.O : s.kind == SEG_DOT ? s.K : (int64_t)s.O * s.K;
}

__device__ inline float seg_element(const Seg& s, int64_t e, const float* w) {
    double acc = 0.0;
    if (s.kind == SEG_SUM) {
        for (int r = 0; r < s.n; ++r) acc += (double)s.rec[(size_t)r * s.stride + s.a + e];
    } else if (s.kind == SEG_DOT) {
        for (int r = 0; r < s.n; ++r) { const float* q = s.rec + (size_t)r * s.stride; acc += (double)q[s.a + e] * (double)q[s.b + e]; }
    } else {
        const int o = (int)(e / s.K), k = (int)(e - (int64_t)o * s.K);
        const bool ln = s.kind == SEG_OUTER_LN;
        const float lw = ln ? w[s.lnw + k] : 1.f, lb = ln ? w[s.lnb + k] : 0.f;
        for (int r = 0; r < s.n; ++r) {
            const float* q = s.rec + (size_t)r * s.stride;
            const float bv = ln ? q[s.b + k] * lw + lb : q[s.b + k];
            acc += (double)q[s.a + o] * (double)bv;
        }
    }
    return (float)acc;
}

__device__ __forceinline__ Seg make_seg(const float* rec, int stride, int n, int kind, int O, int K, int a, int b, int64_t w,
                                        int64_t lnw = 0, int64_t lnb = 0) {
    Seg s;
    s.rec = rec; s.stride = stride; s.n = n; s.kind = kind; s.O = O; s.K = K; s.a = a; s.b = b; s.w = w; s.lnw = lnw; s.lnb = lnb;
    return s;
}

// derivative of act_fn from its output, as torch's backward takes it: relu (y > 0), leaky_relu (y > 0 ? 1 : slope), tanh 1 - y^2
__device__ __forceinline__ float act_grad(float y, int kind) {
    if (kind == 0) return y > 0.f ? 1.f : 0.f;
    if (kind == 1) return y > 0.f ? 1.f : 0.01f;
    return 1.f - y * y;
}

// warp_layer_norm that also keeps x-hat (in `xh`, lane-strided like buf); buf becomes x-hat w + b, the same bits
__device__ __forceinline__ void warp_layer_norm_keep(float* buf, int n, const float* w, const float* b, float* xh, int lane) {
    float s = 0.f;
    for (int k = lane; k < n; k += 32) s += buf[k];
    const float mean = warp_sum(s) / (float)n;
    float q = 0.f;
    for (int k = lane; k < n; k += 32) { const float d = buf[k] - mean; q += d * d; }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)n + LN_EPS);
    for (int k = lane; k < n; k += 32) { const float x = (buf[k] - mean) * rstd; xh[k] = x; buf[k] = x * w[k] + b[k]; }
    __syncwarp();
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// LayerNorm backward (biased variance): dx = rstd (dy w - mean(dy w) - x-hat mean(dy w x-hat)), in f64 with x-hat and rstd taken
// again from the input x = [x0 (n0 values) | x1 (n - n0 values; nullptr: zeros)].  The terms nearly cancel when the LayerNorm is
// narrow (over two values dx is proportional to 1 - x-hat^2 = eps / (var + eps)), so an fp32 x-hat would lose most of dx's digits.
// dy, dx lane-strided.
__device__ __forceinline__ void warp_layer_norm_grad(const float* dy, const float* x0, const float* x1, int n0, int n, const float* w,
                                                     float* dx, int lane) {
    auto x = [&](int k) { return (double)(k < n0 ? x0[k] : (x1 ? x1[k - n0] : 0.f)); };
    double s = 0.0;
    for (int k = lane; k < n; k += 32) s += x(k);
    const double mean = warp_sum_d(s) / n;
    double q = 0.0;
    for (int k = lane; k < n; k += 32) { const double d = x(k) - mean; q += d * d; }
    const double rstd = 1.0 / sqrt(warp_sum_d(q) / n + 1e-5);
    double s1 = 0.0, s2 = 0.0;
    for (int k = lane; k < n; k += 32) { const double g = (double)dy[k] * w[k]; s1 += g; s2 += g * (x(k) - mean) * rstd; }
    s1 = warp_sum_d(s1) / n; s2 = warp_sum_d(s2) / n;
    for (int k = lane; k < n; k += 32) dx[k] = (float)(rstd * ((double)dy[k] * w[k] - s1 - (x(k) - mean) * rstd * s2));
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// position i of a batch of n rows shuffled by `key`: a four-round Feistel network keyed by splitmix64 over the smallest even
// power of two >= n, cycle-walked into [0, n) -- a permutation, computed per row with no table
__device__ __forceinline__ int32_t shuffle_pos(unsigned long long key, int32_t i, int32_t n) {
    if (n <= 1) return i;
    const int bits = 32 - __clz(n - 1), h = (bits + 1) / 2;
    const uint32_t mask = (1u << h) - 1u;
    uint32_t x = (uint32_t)i;
    do {
        uint32_t L = x >> h, R = x & mask;
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const uint32_t F = (uint32_t)splitmix64(key ^ ((unsigned long long)r << 40) ^ R) & mask;
            const uint32_t t = L ^ F; L = R; R = t;
        }
        x = (L << h) | R;
    } while (x >= (uint32_t)n);
    return (int32_t)x;
}

struct GradArgs {
    int32_t mb, start;                   // rows of the launch; the first batch position they take
    const int32_t* n_rows;               // rows in the batch (device)
    int32_t shuffle; unsigned long long key;
    // the batch: full graph features, or the environment's dynamic features + the job type's static ones
    const float* graph_features; const float* obs_dyn; const float* graph_static; const int32_t* model; const uint8_t* mask;
    const float* emb;
    const float* grad_logits; const float* grad_value;              // given upstream gradient (ramp_policy_backward), or
    const int32_t* action; const float* old_logits; const float* adv; const float* vt;     // PPO's (old_logits != nullptr)
    float clip, vf_clip, vf_coeff, ent_coeff, kl_coeff;
    int32_t impala;                      // IMPALA's VTraceLoss instead: adv is pg_adv, vt is vs (old_logits unused)
    int32_t pg;                          // PG's loss instead: adv is the discounted return (old_logits, vt unused)
    float* rec; int32_t* row_model; float* row_stats;               // [mb][..] outputs
    float* logp_old;                     // [batch] log-probability of the action under the old logits, or nullptr
};

__global__ void __launch_bounds__(256) ramp_policy_head_grad_kernel(const PolicyDev P, const GradArgs g) {
    __shared__ float s_x[LRN_WARPS][POL_MAX_DIM], s_f[LRN_WARPS][POL_MAX_DIM], s_d[LRN_WARPS][POL_MAX_DIM];
    __shared__ float s_dh[LRN_WARPS][32 * POL_MAX_HPL], s_dhv[LRN_WARPS][32 * POL_MAX_HPL];
    const ramp_policy_config_t& c = P.c;
    const int gin = c.in_features_graph + c.n_actions, og = c.out_features_graph, on = c.out_features_node, fin = on + og;
    const int H = c.fcnet_hidden, A = c.n_actions, hpl = H / 32, fa = c.fcnet_activation;
    const HeadRec R = head_rec(c);
    const float* w = P.w;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * LRN_WARPS + warp;
    if (i >= g.mb) return;
    float* rec = g.rec + (size_t)i * R.stride;
    const int n = *g.n_rows, pos = g.start + i;
    const int b = pos < n ? (g.shuffle ? shuffle_pos(g.key, pos, n) : pos) : -1;
    const int m = b >= 0 ? g.model[b] : -1;
    if (m < 0 || m >= c.n_models) {                                 // contributes nothing
        for (int k = lane; k < R.stride; k += 32) rec[k] = 0.f;
        if (lane < RS_N) g.row_stats[(size_t)i * RS_N + lane] = 0.f;
        if (lane == 0) g.row_model[i] = -1;
        return;
    }
    float* xb = s_x[warp]; float* fb = s_f[warp]; float* db = s_d[warp];
    // ---- forward: ramp_policy_head_kernel's arithmetic ----
    for (int k = lane; k < gin; k += 32) {
        float x;
        if (k >= c.in_features_graph) x = g.mask[(size_t)b * A + (k - c.in_features_graph)] ? 1.f : 0.f;
        else if (g.graph_features) x = g.graph_features[(size_t)b * c.in_features_graph + k];
        else if (k < 9) x = g.obs_dyn[(size_t)b * 11 + k];
        else if (k < 15) x = g.graph_static[(size_t)m * 6 + (k - 9)];
        else x = g.obs_dyn[(size_t)b * 11 + (k - 6)];
        xb[k] = x;
    }
    __syncwarp();
    warp_layer_norm_keep(xb, gin, w + P.gln_w, w + P.gln_b, rec + R.xg, lane);
    for (int k = lane; k < on; k += 32) fb[k] = g.emb[(size_t)m * on + k];
    if (lane < og) {
        float gg = w[P.gb + lane];
        const float* row = w + P.gW + (size_t)lane * gin;
        for (int k = 0; k < gin; ++k) gg += row[k] * xb[k];
        fb[on + lane] = gg;
    }
    __syncwarp();
    for (int k = lane; k < fin; k += 32) rec[R.fb + k] = fb[k];
    float h[POL_MAX_HPL], hv[POL_MAX_HPL];
#pragma unroll
    for (int u = 0; u < POL_MAX_HPL; ++u) {
        if (u < hpl) {
            const int j = lane + 32 * u;
            float p = w[P.hb + j], q = w[P.vhb + j];
            const float* hr = w + P.hW + (size_t)j * fin; const float* vr = w + P.vhW + (size_t)j * fin;
            for (int k = 0; k < fin; ++k) { const float f = fb[k]; p += hr[k] * f; q += vr[k] * f; }
            h[u] = act_fn(p, fa); hv[u] = act_fn(q, fa);
        }
    }
    float my_logit = -FLT_MAX;
    for (int o = 0; o < A; ++o) {
        float p = 0.f;
#pragma unroll
        for (int u = 0; u < POL_MAX_HPL; ++u) if (u < hpl) p += h[u] * w[P.lW + (size_t)o * H + lane + 32 * u];
        p = warp_sum(p) + w[P.lb + o];
        if (c.apply_action_mask && !g.mask[(size_t)b * A + o]) p += -FLT_MAX;
        if (lane == o) my_logit = p;
    }
    float val = 0.f;
#pragma unroll
    for (int u = 0; u < POL_MAX_HPL; ++u) if (u < hpl) val += hv[u] * w[P.vW + lane + 32 * u];
    val = warp_sum(val) + w[P.vb];
    const float best = warp_max(my_logit);
    const float ex = lane < A ? expf(my_logit - best) : 0.f;
    const float denom = warp_sum(ex);
    const float lp = lane < A ? my_logit - best - logf(denom) : 0.f;      // log-softmax, as act's log-probability
    // ---- upstream gradient: d logits (lane o) and d value ----
    float dl = 0.f, dv = 0.f;
    if (g.impala) {
        // VTraceLoss (impala_torch_policy.py) on one row, summed, not averaged: -logp(a) pg_adv + vf_coeff 0.5 (V - vs)^2
        // - ent_coeff H(pi), with vs and pg_adv constants.  A masked action has probability 0 and adds exactly 0.
        const float pr = ex / denom;
        const int act = g.action[b];
        const float lp_a = __shfl_sync(0xffffffffu, lp, act);
        const float pga = g.adv[b], dvv = val - g.vt[b];
        const float ent = -warp_sum(pr > 0.f ? pr * lp : 0.f);
        if (lane < A) dl = -pga * ((lane == act ? 1.f : 0.f) - pr) + g.ent_coeff * pr * (lp + ent);
        dv = g.vf_coeff * dvv;
        if (lane == 0) {
            float* rs = g.row_stats + (size_t)i * RS_N;
            rs[RS_PI] = -lp_a * pga; rs[RS_VF] = 0.5f * dvv * dvv; rs[RS_ENT] = ent; rs[RS_KL] = 0.f; rs[RS_CLIP] = 0.f;
        }
    } else if (g.pg) {
        // PGTorchPolicy's loss (pg_torch_policy.py): -mean(logp(a) adv) over the batch's rows, no value term.  A masked action
        // has probability 0 and gets exactly 0.  The row's statistics are log p(a) and H(pi), for reporting only.
        const float inv_n = 1.0f / (float)min(g.mb, n - g.start);
        const float pr = ex / denom;
        const int act = g.action[b];
        const float lp_a = __shfl_sync(0xffffffffu, lp, act);
        const float gs = g.adv[b] * inv_n;
        const float ent = -warp_sum(pr > 0.f ? pr * lp : 0.f);
        if (lane < A) dl = -gs * ((lane == act ? 1.f : 0.f) - pr);
        if (lane == 0) {
            float* rs = g.row_stats + (size_t)i * RS_N;
            rs[RS_PI] = lp_a; rs[RS_VF] = 0.f; rs[RS_ENT] = ent; rs[RS_KL] = 0.f; rs[RS_CLIP] = 0.f;
            if (g.logp_old) g.logp_old[b] = lp_a;
        }
    } else if (!g.old_logits) {
        if (lane < A) dl = g.grad_logits[(size_t)b * A + lane];
        dv = g.grad_value[b];
    } else {
        // PPOTorchPolicy.loss (ppo_torch_policy.py) on one row, divided by the minibatch's rows (reduce_mean_valid).  A masked
        // action has probability 0 under both distributions, so it adds exactly 0 to the entropy, the KL and the gradient.
        const float inv_n = 1.0f / (float)min(g.mb, n - g.start);
        const float ol = lane < A ? g.old_logits[(size_t)b * A + lane] : -FLT_MAX;
        const float obest = warp_max(ol);
        const float oex = lane < A ? expf(ol - obest) : 0.f;
        const float oden = warp_sum(oex);
        const float olp = lane < A ? ol - obest - logf(oden) : 0.f;
        const float pr = ex / denom, oq = oex / oden;
        const int act = g.action[b];
        const float lp_a = __shfl_sync(0xffffffffu, lp, act), olp_a = __shfl_sync(0xffffffffu, olp, act);
        const float ratio = expf(lp_a - olp_a);
        const float adv = g.adv[b];
        const float s1 = adv * ratio, s2 = adv * fminf(fmaxf(ratio, 1.f - g.clip), 1.f + g.clip);
        const bool cut = s2 < s1;        // min() takes the clipped term: no gradient through the ratio
        const float ent = -warp_sum(pr > 0.f ? pr * lp : 0.f);
        const float kl = warp_sum(oq > 0.f ? oq * (olp - lp) : 0.f);
        const float dvv = val - g.vt[b], vf = dvv * dvv;
        const float gs = cut ? 0.f : adv * ratio;                   // d min(..) / d logp(a)
        if (lane < A) dl = inv_n * (-gs * ((lane == act ? 1.f : 0.f) - pr) + g.ent_coeff * pr * (lp + ent) + g.kl_coeff * (pr - oq));
        dv = vf <= g.vf_clip ? inv_n * g.vf_coeff * 2.f * dvv : 0.f;
        if (lane == 0) {
            float* rs = g.row_stats + (size_t)i * RS_N;
            rs[RS_PI] = -fminf(s1, s2); rs[RS_VF] = fminf(vf, g.vf_clip); rs[RS_ENT] = ent; rs[RS_KL] = kl; rs[RS_CLIP] = cut ? 1.f : 0.f;
            if (g.logp_old) g.logp_old[b] = olp_a;
        }
    }
    if (lane < A) rec[R.dl + lane] = dl;
    if (lane == 0) { rec[R.dv] = dv; g.row_model[i] = m; }
    // ---- logits / value layers -> hidden pre-activations ----
    if (lane < A) db[lane] = dl;
    __syncwarp();
    float* dhs = s_dh[warp]; float* dvs = s_dhv[warp];
#pragma unroll
    for (int u = 0; u < POL_MAX_HPL; ++u) {
        if (u < hpl) {
            const int j = lane + 32 * u;
            float d = 0.f;
            for (int o = 0; o < A; ++o) d += db[o] * w[P.lW + (size_t)o * H + j];
            const float dp = d * act_grad(h[u], fa), dq = dv * w[P.vW + j] * act_grad(hv[u], fa);
            dhs[j] = dp; dvs[j] = dq;
            rec[R.h + j] = h[u]; rec[R.hv + j] = hv[u]; rec[R.dh + j] = dp; rec[R.dhv + j] = dq;
        }
    }
    __syncwarp();
    // ---- hidden layers -> read-out input [emb | graph module] ----
    for (int k = lane; k < fin; k += 32) {
        float d = 0.f;
        for (int j = 0; j < H; ++j) d += w[P.hW + (size_t)j * fin + k] * dhs[j] + w[P.vhW + (size_t)j * fin + k] * dvs[j];
        db[k] = d;
    }
    __syncwarp();
    for (int k = lane; k < on; k += 32) rec[R.de + k] = db[k];
    // ---- graph module Linear -> its LayerNorm output (the input [graph features | mask] is data: no gradient) ----
    if (lane < og) rec[R.dpg + lane] = db[on + lane];
    for (int k = lane; k < gin; k += 32) {
        float d = 0.f;
        for (int o = 0; o < og; ++o) d += w[P.gW + (size_t)o * gin + k] * db[on + o];
        rec[R.dyg + k] = d;
    }
}

// the read-out's and graph module's segments in blob order (host: the learner's setup)
inline int head_segs(const PolicyDev& P, const float* rec, int mb, Seg* s) {
    const ramp_policy_config_t& c = P.c;
    const HeadRec R = head_rec(c);
    const int gin = c.in_features_graph + c.n_actions, og = c.out_features_graph, fin = c.out_features_node + og, H = c.fcnet_hidden, A = c.n_actions;
    auto seg = [&](int kind, int O, int K, int a, int b, int64_t w, int64_t lnw = 0, int64_t lnb = 0) {
        Seg x; x.rec = rec; x.stride = R.stride; x.n = mb; x.kind = kind; x.O = O; x.K = K; x.a = a; x.b = b; x.w = w; x.lnw = lnw; x.lnb = lnb;
        return x;
    };
    int k = 0;
    s[k++] = seg(SEG_DOT, 0, gin, R.dyg, R.xg, P.gln_w);
    s[k++] = seg(SEG_SUM, gin, 0, R.dyg, 0, P.gln_b);
    s[k++] = seg(SEG_OUTER_LN, og, gin, R.dpg, R.xg, P.gW, P.gln_w, P.gln_b);
    s[k++] = seg(SEG_SUM, og, 0, R.dpg, 0, P.gb);
    s[k++] = seg(SEG_OUTER, H, fin, R.dh, R.fb, P.hW);
    s[k++] = seg(SEG_SUM, H, 0, R.dh, 0, P.hb);
    s[k++] = seg(SEG_OUTER, A, H, R.dl, R.h, P.lW);
    s[k++] = seg(SEG_SUM, A, 0, R.dl, 0, P.lb);
    s[k++] = seg(SEG_OUTER, H, fin, R.dhv, R.fb, P.vhW);
    s[k++] = seg(SEG_SUM, H, 0, R.dhv, 0, P.vhb);
    s[k++] = seg(SEG_OUTER, 1, H, R.dv, R.hv, P.vW);
    s[k++] = seg(SEG_SUM, 1, 0, R.dv, 0, P.vb);
    return k;
}
constexpr int HEAD_SEGS = 12;

__global__ void __launch_bounds__(256) ramp_policy_head_reduce_kernel(const PolicyDev P, const Seg* segs, int32_t n_segs, int64_t total, float* grad) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        int si = 0;
        int64_t off = e;
        while (si + 1 < n_segs && off >= seg_size(segs[si])) { off -= seg_size(segs[si]); ++si; }
        grad[segs[si].w + off] = seg_element(segs[si], off, P.w);
    }
}

// per job type: the rounds' node states and module outputs, kept for the backward, and its records (ramp_policy_learn's scratch)
struct GradModelDev {
    const int32_t* out_ptr; const int32_t* out_edge;   // CSR by source node, in edge order (ramp_policy_set_model)
    float* z;                            // [num_rounds][N][zs]   output of every round
    float* hn; float* he;                // [num_rounds][N][msg/2], [num_rounds][E][msg/2]
    float* dz; float* dz2;               // [N][zs]               d round output, d round input
    float* dhn;                          // [N][msg/2]
    float* nrec; float* erec; float* mrec;   // node / edge / reduce-module items: [x-hat | d LN output | d Linear output]
    float* mdx;                          // [N + E][msg]          d reduce-module input per item (own state: item v; edge e: N + e)
};

struct GnnDims { int32_t zs, zin, zout, nrs, ers, mrs; };   // widest round input / output, record strides

__host__ __device__ inline GnnDims gnn_dims(const ramp_policy_config_t& c) {
    GnnDims d;
    const int half = c.out_features_msg / 2;
    d.zin = c.in_features_node > c.out_features_hidden ? c.in_features_node : c.out_features_hidden;
    d.zout = c.out_features_node > c.out_features_hidden ? c.out_features_node : c.out_features_hidden;
    d.zs = d.zin > d.zout ? d.zin : d.zout;
    d.nrs = 2 * d.zin + half; d.ers = 2 * c.in_features_edge + half; d.mrs = 2 * c.out_features_msg + d.zout;
    return d;
}

// ramp_gnn_embed_grad_kernel runs in two launches around the head gradient: EMB_FORWARD runs the MeanPool rounds and keeps every
// round's states (and writes the embeddings when `emb` is given: ramp_gnn_embed_kernel's arithmetic, the same bits), EMB_BACKWARD
// runs backward from them.  A forward for a minibatch past the batch's end does nothing: no update ran, the kept states are current.
enum { EMB_FORWARD = 1, EMB_BACKWARD = 2 };
struct EmbGradArgs {
    const int32_t* n_rows; int32_t start;                           // forward: the batch's rows (device, or nullptr) and the minibatch
    float* emb;                                                     // forward: [n_models][out_node] or nullptr
    const float* rec; const int32_t* row_model; int32_t rows;       // backward: the head-gradient kernel's records
    float* gpart; int64_t n_gnn;                                    // backward: [n_models][n_gnn] per job type gradients of the rounds' weights
};

template <int MODE>
__global__ void __launch_bounds__(256, 1) ramp_gnn_embed_grad_kernel(const PolicyDev P, const ModelDev* models, const GradModelDev* gms, const EmbGradArgs g) {
    __shared__ float s_a[8][POL_MAX_DIM], s_b[8][POL_MAX_DIM], s_demb[POL_MAX_DIM];
    const ramp_policy_config_t& c = P.c;
    const int m = blockIdx.x;
    const ModelDev M = models[m];
    const GradModelDev G = gms[m];
    const GnnDims D = gnn_dims(c);
    const HeadRec HR = head_rec(c);
    float* part = g.gpart + (size_t)m * g.n_gnn;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
    const int on = c.out_features_node, msg = c.out_features_msg, half = msg / 2, ine = c.in_features_edge, ak = c.aggregator_activation;
    const int N = M.n_nodes, E = M.n_edges;
    const float* w = P.w;
    if (MODE == EMB_BACKWARD) {
        // ---- d emb[m]: the rows of this job type, in row order ----
        int any = 0;
        for (int k = threadIdx.x; k < on; k += blockDim.x) {
            double s = 0.0;
            for (int r = 0; r < g.rows; ++r) if (g.row_model[r] == m) s += (double)g.rec[(size_t)r * HR.stride + HR.de + k];
            s_demb[k] = (float)s;
            any |= s != 0.0;
        }
        if (!__syncthreads_or(any) || N <= 0) {
            for (int64_t e = threadIdx.x; e < g.n_gnn; e += blockDim.x) part[e] = 0.f;
            return;
        }
    } else if (N <= 0 || (g.n_rows && g.start >= *g.n_rows)) {
        return;
    }
    float* buf = s_a[warp];
    float* dp = s_b[warp];
    auto zin_of = [&](int r) { return r == 0 ? M.nf : G.z + (size_t)(r - 1) * N * D.zs; };
    // ---- forward: ramp_gnn_embed_kernel's rounds, every round's output and module outputs kept ----
    for (int r = 0; r < c.num_rounds && MODE == EMB_FORWARD; ++r) {
        const RoundW R = P.rounds[r];
        const float* zin = zin_of(r);
        const int zst = r == 0 ? c.in_features_node : D.zs;
        float* zout = G.z + (size_t)r * N * D.zs;
        float* hn = G.hn + (size_t)r * N * half;
        float* he = G.he + (size_t)r * E * half;
        for (int v = warp; v < N; v += n_warps) {
            for (int k = lane; k < R.in; k += 32) buf[k] = zin[(size_t)v * zst + k];
            __syncwarp();
            warp_layer_norm(buf, R.in, w + R.nln_w, w + R.nln_b, lane);
            for (int o = lane; o < half; o += 32) {
                float a = w[R.nb + o];
                const float* row = w + R.nW + (size_t)o * R.in;
                for (int k = 0; k < R.in; ++k) a += row[k] * buf[k];
                hn[(size_t)v * half + o] = act_fn(a, ak);
            }
            __syncwarp();
        }
        for (int e = warp; e < E; e += n_warps) {
            for (int k = lane; k < ine; k += 32) buf[k] = M.ef[(size_t)e * ine + k];
            __syncwarp();
            warp_layer_norm(buf, ine, w + R.eln_w, w + R.eln_b, lane);
            for (int o = lane; o < half; o += 32) {
                float a = w[R.eb + o];
                const float* row = w + R.eW + (size_t)o * ine;
                for (int k = 0; k < ine; ++k) a += row[k] * buf[k];
                he[(size_t)e * half + o] = act_fn(a, ak);
            }
            __syncwarp();
        }
        __syncthreads();
        for (int v = warp; v < N; v += n_warps) {
            const int e0 = M.in_ptr[v], e1 = M.in_ptr[v + 1];
            float acc[POL_MAX_DIM / 32];
#pragma unroll
            for (int q = 0; q < POL_MAX_DIM / 32; ++q) acc[q] = 0.f;
            if (e1 > e0) {
                for (int mi = -1; mi < e1 - e0; ++mi) {
                    const int src = mi < 0 ? v : M.in_src[e0 + mi];
                    for (int k = lane; k < half; k += 32) {
                        buf[k] = hn[(size_t)src * half + k];
                        buf[half + k] = mi < 0 ? 0.f : he[(size_t)M.in_edge[e0 + mi] * half + k];
                    }
                    __syncwarp();
                    warp_layer_norm(buf, msg, w + R.rln_w, w + R.rln_b, lane);
#pragma unroll
                    for (int q = 0; q < POL_MAX_DIM / 32; ++q) {
                        const int o = lane + 32 * q;
                        if (o < R.out) {
                            float a = w[R.rb + o];
                            const float* row = w + R.rW + (size_t)o * msg;
                            for (int k = 0; k < msg; ++k) a += row[k] * buf[k];
                            acc[q] += act_fn(a, ak);
                        }
                    }
                    __syncwarp();
                }
            }
            const float inv = 1.0f / (float)(e1 - e0 + 1);
#pragma unroll
            for (int q = 0; q < POL_MAX_DIM / 32; ++q) {
                const int o = lane + 32 * q;
                if (o < R.out) zout[(size_t)v * D.zs + o] = acc[q] * inv;
            }
        }
        __syncthreads();
    }
    if (MODE == EMB_FORWARD) {
        if (g.emb) {                                                // the mean over the job's nodes, as ramp_gnn_embed_kernel takes it
            const float* zl = zin_of(c.num_rounds);
            for (int o = threadIdx.x; o < on; o += blockDim.x) {
                float s = 0.f;
                for (int v = 0; v < N; ++v) s += zl[(size_t)v * D.zs + o];
                g.emb[(size_t)m * on + o] = s / (float)N;
            }
        }
        return;
    }
    // ---- backward: d of the last round's output is d emb / n_nodes at every node (the node mean) ----
    float* dz = G.dz; float* dzin = G.dz2;
    for (int64_t x = threadIdx.x; x < (int64_t)N * on; x += blockDim.x) {
        const int v = (int)(x / on), k = (int)(x - (int64_t)v * on);
        dz[(size_t)v * D.zs + k] = s_demb[k] / (float)N;
    }
    __syncthreads();
    for (int r = c.num_rounds - 1; r >= 0; --r) {
        const RoundW R = P.rounds[r];
        const float* zin = zin_of(r);
        const int zst = r == 0 ? c.in_features_node : D.zs;
        const float* hn = G.hn + (size_t)r * N * half;
        const float* he = G.he + (size_t)r * E * half;
        // reduce module, per destination node: its own state (item v) and every incoming message (item N + e), each scaled by
        // 1 / (deg + 1); a zero-in-degree node's output is the constant 0, so its items carry nothing
        for (int v = warp; v < N; v += n_warps) {
            const int e0 = M.in_ptr[v], e1 = M.in_ptr[v + 1];
            if (e1 == e0) {
                float* rr = G.mrec + (size_t)v * D.mrs;
                for (int k = lane; k < D.mrs; k += 32) rr[k] = 0.f;
                for (int k = lane; k < msg; k += 32) G.mdx[(size_t)v * msg + k] = 0.f;
                continue;
            }
            const float inv = 1.0f / (float)(e1 - e0 + 1);
            for (int mi = -1; mi < e1 - e0; ++mi) {
                const int src = mi < 0 ? v : M.in_src[e0 + mi];
                const int item = mi < 0 ? v : N + M.in_edge[e0 + mi];
                float* rr = G.mrec + (size_t)item * D.mrs;
                for (int k = lane; k < half; k += 32) {
                    buf[k] = hn[(size_t)src * half + k];
                    buf[half + k] = mi < 0 ? 0.f : he[(size_t)M.in_edge[e0 + mi] * half + k];
                }
                __syncwarp();
                warp_layer_norm_keep(buf, msg, w + R.rln_w, w + R.rln_b, rr, lane);
                for (int o = lane; o < R.out; o += 32) {
                    float a = w[R.rb + o];
                    const float* row = w + R.rW + (size_t)o * msg;
                    for (int k = 0; k < msg; ++k) a += row[k] * buf[k];
                    const float d = dz[(size_t)v * D.zs + o] * inv * act_grad(act_fn(a, ak), ak);
                    dp[o] = d; rr[2 * msg + o] = d;
                }
                __syncwarp();
                for (int k = lane; k < msg; k += 32) {
                    float d = 0.f;
                    for (int o = 0; o < R.out; ++o) d += w[R.rW + (size_t)o * msg + k] * dp[o];
                    rr[msg + k] = d;
                }
                warp_layer_norm_grad(rr + msg, hn + (size_t)src * half, mi < 0 ? nullptr : he + (size_t)M.in_edge[e0 + mi] * half, half, msg,
                                     w + R.rln_w, G.mdx + (size_t)item * msg, lane);
                __syncwarp();
            }
        }
        __syncthreads();
        // d node-module output: the node's own state plus what its messages received, gathered by source
        for (int64_t x = threadIdx.x; x < (int64_t)N * half; x += blockDim.x) {
            const int u = (int)(x / half), k = (int)(x - (int64_t)u * half);
            float s = G.mdx[(size_t)u * msg + k];
            for (int q = G.out_ptr[u]; q < G.out_ptr[u + 1]; ++q) s += G.mdx[(size_t)(N + G.out_edge[q]) * msg + k];
            G.dhn[(size_t)u * half + k] = s;
        }
        __syncthreads();
        // node module -> the round's input (the previous round's output), edge module (its input is data)
        for (int u = warp; u < N; u += n_warps) {
            float* rr = G.nrec + (size_t)u * D.nrs;
            for (int k = lane; k < R.in; k += 32) buf[k] = zin[(size_t)u * zst + k];
            __syncwarp();
            warp_layer_norm_keep(buf, R.in, w + R.nln_w, w + R.nln_b, rr, lane);
            for (int o = lane; o < half; o += 32) {
                const float d = G.dhn[(size_t)u * half + o] * act_grad(hn[(size_t)u * half + o], ak);
                dp[o] = d; rr[2 * D.zin + o] = d;
            }
            __syncwarp();
            for (int k = lane; k < R.in; k += 32) {
                float d = 0.f;
                for (int o = 0; o < half; ++o) d += w[R.nW + (size_t)o * R.in + k] * dp[o];
                rr[D.zin + k] = d;
            }
            if (r > 0) warp_layer_norm_grad(rr + D.zin, zin + (size_t)u * zst, nullptr, R.in, R.in, w + R.nln_w, dzin + (size_t)u * D.zs, lane);
            __syncwarp();
        }
        for (int e = warp; e < E; e += n_warps) {
            float* rr = G.erec + (size_t)e * D.ers;
            for (int k = lane; k < ine; k += 32) buf[k] = M.ef[(size_t)e * ine + k];
            __syncwarp();
            warp_layer_norm_keep(buf, ine, w + R.eln_w, w + R.eln_b, rr, lane);
            for (int o = lane; o < half; o += 32) {
                const float d = G.mdx[(size_t)(N + e) * msg + half + o] * act_grad(he[(size_t)e * half + o], ak);
                dp[o] = d; rr[2 * ine + o] = d;
            }
            __syncwarp();
            for (int k = lane; k < ine; k += 32) {
                float d = 0.f;
                for (int o = 0; o < half; ++o) d += w[R.eW + (size_t)o * ine + k] * dp[o];
                rr[ine + k] = d;
            }
            __syncwarp();
        }
        __syncthreads();
        // this round's weight gradients: every element a sum over the items in order
        for (int si = 0; si < 12; ++si) {
            Seg s;
            const int mod = si / 4, part_i = si % 4;
            if (mod == 0) {
                const int in = R.in;
                s = part_i == 0 ? make_seg(G.nrec, D.nrs, N, SEG_DOT, 0, in, D.zin, 0, R.nln_w)
                  : part_i == 1 ? make_seg(G.nrec, D.nrs, N, SEG_SUM, in, 0, D.zin, 0, R.nln_b)
                  : part_i == 2 ? make_seg(G.nrec, D.nrs, N, SEG_OUTER_LN, half, in, 2 * D.zin, 0, R.nW, R.nln_w, R.nln_b)
                  : make_seg(G.nrec, D.nrs, N, SEG_SUM, half, 0, 2 * D.zin, 0, R.nb);
            } else if (mod == 1) {
                s = part_i == 0 ? make_seg(G.erec, D.ers, E, SEG_DOT, 0, ine, ine, 0, R.eln_w)
                  : part_i == 1 ? make_seg(G.erec, D.ers, E, SEG_SUM, ine, 0, ine, 0, R.eln_b)
                  : part_i == 2 ? make_seg(G.erec, D.ers, E, SEG_OUTER_LN, half, ine, 2 * ine, 0, R.eW, R.eln_w, R.eln_b)
                  : make_seg(G.erec, D.ers, E, SEG_SUM, half, 0, 2 * ine, 0, R.eb);
            } else {
                s = part_i == 0 ? make_seg(G.mrec, D.mrs, N + E, SEG_DOT, 0, msg, msg, 0, R.rln_w)
                  : part_i == 1 ? make_seg(G.mrec, D.mrs, N + E, SEG_SUM, msg, 0, msg, 0, R.rln_b)
                  : part_i == 2 ? make_seg(G.mrec, D.mrs, N + E, SEG_OUTER_LN, R.out, msg, 2 * msg, 0, R.rW, R.rln_w, R.rln_b)
                  : make_seg(G.mrec, D.mrs, N + E, SEG_SUM, R.out, 0, 2 * msg, 0, R.rb);
            }
            const int64_t sz = seg_size(s);
            for (int64_t e = threadIdx.x; e < sz; e += blockDim.x) part[s.w + e] = seg_element(s, e, w);
        }
        __syncthreads();
        float* t = dz; dz = dzin; dzin = t;
    }
}

// block-wide sum in a fixed order (every thread gets it)
__device__ __forceinline__ double block_sum(double v, double* s_red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0) s_red[warp] = v;
    __syncthreads();
    double t = lane < nw ? s_red[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    return t;
}

__global__ void __launch_bounds__(256) ramp_grad_finish_kernel(const float* gpart, int32_t n_models, int64_t n_gnn, int64_t n_w, float* grad, double* norm_part) {
    __shared__ double s_red[32];
    double q = 0.0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_w; e += (int64_t)gridDim.x * blockDim.x) {
        float v;
        if (e < n_gnn) {
            double s = 0.0;
            for (int m = 0; m < n_models; ++m) s += (double)gpart[(size_t)m * n_gnn + e];
            v = (float)s;
            grad[e] = v;
        } else {
            v = grad[e];
        }
        q += (double)v * (double)v;
    }
    q = block_sum(q, s_red);
    if (threadIdx.x == 0) norm_part[blockIdx.x] = q;
}

// the minibatch's statistics (RAMP_PPO_*): means over its rows, and the gradient's global norm before clipping
__device__ inline void minibatch_stats(const float* row_stats, int rows, float vf_coeff, float ent_coeff, float kl_coeff, double norm, double* out) {
    double s[RS_N] = {0, 0, 0, 0, 0};
    for (int r = 0; r < rows; ++r)
        for (int k = 0; k < RS_N; ++k) s[k] += (double)row_stats[(size_t)r * RS_N + k];
    for (int k = 0; k < RS_N; ++k) s[k] /= (double)rows;
    out[RAMP_PPO_TOTAL_LOSS] = s[RS_PI] + (double)vf_coeff * s[RS_VF] - (double)ent_coeff * s[RS_ENT] + (double)kl_coeff * s[RS_KL];
    out[RAMP_PPO_POLICY_LOSS] = s[RS_PI]; out[RAMP_PPO_VF_LOSS] = s[RS_VF]; out[RAMP_PPO_ENTROPY] = s[RS_ENT];
    out[RAMP_PPO_KL] = s[RS_KL]; out[RAMP_PPO_CLIP_FRAC] = s[RS_CLIP]; out[RAMP_PPO_GRAD_NORM] = norm;
    out[RAMP_PPO_KL_COEFF] = kl_coeff; out[RAMP_PPO_ROWS] = rows;
}

__device__ __forceinline__ double sum_norm_parts(const double* norm_part) {
    double s = 0.0;
    for (int k = 0; k < LRN_GRID; ++k) s += norm_part[k];
    return sqrt(s);
}

// torch.optim.Adam takes its hyper-parameters as Python floats: the bias corrections and the step size in double, and each
// per-element scalar (beta2, 1 - beta1, 1 - beta2 -- formed in double --, eps, -step_size) rounded to fp32 once
struct AdamArgs {
    double lr, beta1, beta2;                 // the bias corrections, in double
    float beta2_f, one_m_beta1, one_m_beta2, eps, max_norm;   // the fp32 scalars; max_norm <= 0: no clipping
    const int32_t* n_rows; int32_t mb, start;
    int32_t* step; int32_t parity;           // Adam's step count: read from step[parity], written to step[parity ^ 1]
    float* m; float* v; float* grad; const double* norm_part; float* w;
    const float* row_stats; float vf_coeff, ent_coeff, kl_coeff; double* stats;   // RAMP_PPO_STATS_LEN for this minibatch
};

__global__ void __launch_bounds__(256) ramp_adam_kernel(const AdamArgs a, int64_t n_w) {
    __shared__ double s_norm;
    const int rows = max(0, min(a.mb, *a.n_rows - a.start));
    const int t0 = a.step[a.parity];
    if (rows == 0) {                                                // past the batch's end: no update
        if (blockIdx.x == 0 && threadIdx.x == 0) { a.step[a.parity ^ 1] = t0; a.stats[RAMP_PPO_ROWS] = 0.0; }
        return;
    }
    const int t = t0 + 1;
    if (threadIdx.x == 0) s_norm = sum_norm_parts(a.norm_part);
    __syncthreads();
    const double norm = s_norm;
    // clip_grad_norm_: coef = min(1, max_norm / (norm + 1e-6)); torch.optim.Adam (betas, eps, bias correction)
    // (torch forms it on the fp32 norm, in fp32)
    const float coef = a.max_norm > 0.f ? fminf(1.f, a.max_norm / ((float)norm + 1e-6f)) : 1.f;
    const double bc1 = 1.0 - pow(a.beta1, (double)t), bc2 = 1.0 - pow(a.beta2, (double)t);
    const float step_size = (float)(a.lr / bc1), bc2_sqrt = (float)sqrt(bc2);
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_w; e += (int64_t)gridDim.x * blockDim.x) {
        const float gr = a.grad[e] * coef;
        const float mm = a.m[e] + a.one_m_beta1 * (gr - a.m[e]);            // exp_avg.lerp_(grad, 1 - beta1)
        const float vv = a.v[e] * a.beta2_f + a.one_m_beta2 * gr * gr;       // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
        a.m[e] = mm; a.v[e] = vv;
        a.w[e] -= step_size * (mm / (sqrtf(vv) / bc2_sqrt + a.eps));
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        a.step[a.parity ^ 1] = t;
        if (a.row_stats) minibatch_stats(a.row_stats, rows, a.vf_coeff, a.ent_coeff, a.kl_coeff, norm, a.stats);
    }
}

// ramp_ppo_loss_grad's statistics (no update)
__global__ void ramp_ppo_minibatch_stats_kernel(const float* row_stats, int32_t rows, float vf_coeff, float ent_coeff, float kl_coeff,
                                                const double* norm_part, double* out) {
    minibatch_stats(row_stats, rows, vf_coeff, ent_coeff, kl_coeff, sum_norm_parts(norm_part), out);
}

// the mean of the last pass's minibatch statistics, and RLlib's PPO update_kl from its mean KL
__global__ void ramp_ppo_learn_stats_kernel(const double* mb_stats, int32_t n_mb, float kl_coeff, float kl_target, const int32_t* n_rows, double* out) {
    double s[RAMP_PPO_STATS_LEN] = {};
    int k = 0;
    for (int i = 0; i < n_mb; ++i) {
        const double* x = mb_stats + (size_t)i * RAMP_PPO_STATS_LEN;
        if (x[RAMP_PPO_ROWS] <= 0.0) continue;
        for (int j = 0; j < RAMP_PPO_STATS_LEN; ++j) s[j] += x[j];
        ++k;
    }
    for (int j = 0; j < RAMP_PPO_STATS_LEN; ++j) out[j] = k ? s[j] / k : 0.0;
    double c = kl_coeff;
    if (k) {
        if (out[RAMP_PPO_KL] > 2.0 * kl_target) c *= 1.5;
        else if (out[RAMP_PPO_KL] < 0.5 * kl_target) c *= 0.5;
    }
    out[RAMP_PPO_KL_COEFF] = c;
    out[RAMP_PPO_ROWS] = *n_rows;
}

struct GaeArgs {
    int32_t T, B, A, n_models, standardize;
    double gamma, lambda;
    const float* t_obs; const int32_t* t_model; const uint8_t* t_mask; const int32_t* t_action; const float* t_logp;
    const float* t_value; const double* t_reward; const uint8_t* t_done;   // t_value nullptr: no critic (PG), V = 0
    const float* boot;                   // [B] value of the state after the last step (unused without t_value)
    double* adv64;                       // [T][B] scratch
    float* obs; int32_t* model; uint8_t* mask; int32_t* action; float* logp; float* adv; float* vt; int32_t* n_rows;   // the batch
};

// one CTA: GAE (RLlib compute_advantages, use_gae) per episode, one thread per episode scanning backwards; then the rows of
// episodes that were not finished when the decision was taken and had a queued job, t-major; then (a - mean) / max(1e-4, std).
// Without values (t_value nullptr, lambda 1) the scan is r_t + gamma (1 - done_t) next with a 0 bootstrap: RLlib's
// compute_advantages(use_gae=False, use_critic=False, last_r=0), discount_cumsum's recursion in f64; value_target = advantage.
__global__ void __launch_bounds__(1024) ramp_ppo_gae_kernel(const GaeArgs a) {
    __shared__ double s_red[32];
    __shared__ int s_scan[32];
    const int T = a.T, B = a.B;
    auto alive = [&](int t, int b) { return t == 0 || !a.t_done[(size_t)(t - 1) * B + b]; };
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        double next = 0.0;
        for (int t = T - 1; t >= 0; --t) {
            const size_t i = (size_t)t * B + b;
            if (!alive(t, b)) { a.adv64[i] = 0.0; continue; }
            const double nonterm = a.t_done[i] ? 0.0 : 1.0;
            const double V = a.t_value ? (double)a.t_value[i] : 0.0;
            const double Vn = !a.t_value ? 0.0 : t == T - 1 ? (double)a.boot[b] : (double)a.t_value[i + B];
            const double delta = a.t_reward[i] + a.gamma * Vn * nonterm - V;
            next = delta + a.gamma * a.lambda * nonterm * next;
            a.adv64[i] = next;
        }
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    int base = 0;
    for (int t = 0; t < T; ++t) {
        for (int b0 = 0; b0 < B; b0 += blockDim.x) {
            const int b = b0 + threadIdx.x;
            const size_t i = (size_t)t * B + b;
            const int flag = b < B && alive(t, b) && a.t_model[i] >= 0 && a.t_model[i] < a.n_models;
            int x = flag;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
            if (lane == 31) s_scan[warp] = x;
            __syncthreads();
            if (warp == 0) {
                int y = lane < nw ? s_scan[lane] : 0;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int z = __shfl_up_sync(0xffffffffu, y, o); if (lane >= o) y += z; }
                s_scan[lane] = y;                                   // inclusive over warps
            }
            __syncthreads();
            const int pos = base + (warp ? s_scan[warp - 1] : 0) + x - flag;
            if (flag) {
                for (int k = 0; k < 11; ++k) a.obs[(size_t)pos * 11 + k] = a.t_obs[i * 11 + k];
                for (int k = 0; k < a.A; ++k) a.mask[(size_t)pos * a.A + k] = a.t_mask[i * a.A + k];
                a.model[pos] = a.t_model[i]; a.action[pos] = a.t_action[i]; a.logp[pos] = a.t_logp[i];
                a.adv[pos] = (float)a.adv64[i];
                a.vt[pos] = (float)(a.adv64[i] + (a.t_value ? (double)a.t_value[i] : 0.0));
            }
            base += s_scan[nw - 1];
            __syncthreads();
        }
    }
    const int n = base;
    for (int64_t i = n + threadIdx.x; i < (int64_t)T * B; i += blockDim.x) a.model[i] = -1;
    if (a.standardize && n > 0) {
        double s = 0.0;
        for (int i = threadIdx.x; i < n; i += blockDim.x) s += a.adv[i];
        const double mean = block_sum(s, s_red) / n;
        double q = 0.0;
        for (int i = threadIdx.x; i < n; i += blockDim.x) { const double d = a.adv[i] - mean; q += d * d; }
        const double sd = fmax(1e-4, sqrt(block_sum(q, s_red) / n));
        for (int i = threadIdx.x; i < n; i += blockDim.x) a.adv[i] = (float)((a.adv[i] - mean) / sd);
    }
    if (threadIdx.x == 0) *a.n_rows = n;
}

// ---- IMPALA (ramp_policy_learn_impala, ramp_impala_loss_grad) ----

struct ImpalaBatchArgs {
    int32_t T, B, A, L, n_models;
    const float* t_obs; const int32_t* t_model; const uint8_t* t_mask; const int32_t* t_action; const float* t_logp;
    const double* t_reward; const uint8_t* t_done;
    float* obs; int32_t* model; uint8_t* mask; int32_t* action; float* blogp; double* reward; uint8_t* done; int32_t* n_rows;
};

// the first T slots of the trajectory as fragments of L rows, fragment f = (time block f / B, episode f % B), row r = f L + t.
// A row whose episode had already finished, or had nothing queued (or a job type outside the policy's), gets model -1.
__global__ void ramp_impala_batch_kernel(const ImpalaBatchArgs a) {
    const int64_t R = (int64_t)a.T * a.B;
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r == 0) *a.n_rows = (int32_t)R;
    if (r >= R) return;
    const int64_t f = r / a.L, t = r - f * a.L, j = f / a.B, b = f - j * a.B;
    const size_t s = (size_t)(j * a.L + t), i = s * a.B + b;
    const bool alive = s == 0 || !a.t_done[i - a.B];
    const int32_t m = a.t_model[i];
    for (int k = 0; k < 11; ++k) a.obs[r * 11 + k] = a.t_obs[i * 11 + k];
    for (int k = 0; k < a.A; ++k) a.mask[r * a.A + k] = a.t_mask[i * a.A + k];
    a.model[r] = alive && m >= 0 && m < a.n_models ? m : -1;
    a.action[r] = a.t_action[i]; a.blogp[r] = a.t_logp[i]; a.reward[r] = a.t_reward[i]; a.done[r] = a.t_done[i];
}

struct VtraceArgs {
    int32_t L, n_frag, row0, A, n_models;
    double gamma, clip_rho, clip_pg_rho;
    const float* logits; const float* value;                        // the head kernel's at the current weights
    const int32_t* model; const int32_t* action; const float* blogp; const double* reward; const uint8_t* done;
    float* tlogp; float* log_rho; float* vs; float* pg_adv; int32_t* lmodel;
};

// one warp per fragment: the target log-probability of every row's action -- the head kernel's log-softmax, operation for
// operation, so at the collection weights it is the collected value bit for bit -- then from_importance_weights (vtrace_torch.py)
// scanning backwards in f64 with vtrace_drop_last_ts: rows 0 .. L-2 are the loss's, row L-1's value is the bootstrap and vs_{L-1}.
// A row without a decision has log rho 0, V 0 (the head kernel's), its reward and done, and stays out of the loss (lmodel -1).
__global__ void __launch_bounds__(256) ramp_vtrace_kernel(const VtraceArgs a) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int f = blockIdx.x * (blockDim.x >> 5) + warp;
    if (f >= a.n_frag) return;
    const int64_t r0 = (int64_t)a.row0 + (int64_t)f * a.L;
    for (int t = 0; t < a.L; ++t) {
        const int64_t r = r0 + t;
        const int m = a.model[r];
        if (m < 0 || m >= a.n_models) {
            if (lane == 0) { a.tlogp[r] = 0.f; a.log_rho[r] = 0.f; }
            continue;
        }
        const float l = lane < a.A ? a.logits[r * a.A + lane] : -FLT_MAX;
        const float best = warp_max(l);
        const float ex = lane < a.A ? expf(l - best) : 0.f;
        const float denom = warp_sum(ex);
        const float chosen = __shfl_sync(0xffffffffu, l, a.action[r]);
        if (lane == 0) {
            const float lp = chosen - best - logf(denom);
            a.tlogp[r] = lp;
            a.log_rho[r] = (float)((double)lp - (double)a.blogp[r]);
        }
    }
    if (lane != 0) return;                                          // lane 0 wrote every row's log-probability above
    const int64_t rl = r0 + a.L - 1;
    const double boot = a.value[rl];
    a.vs[rl] = (float)boot; a.pg_adv[rl] = 0.f; a.lmodel[rl] = -1;
    double v_next = boot, vs_next = boot, acc = 0.0;                // acc: vs_{t+1} - V_{t+1}
    for (int t = a.L - 2; t >= 0; --t) {
        const int64_t r = r0 + t;
        const int m = a.model[r];
        const bool valid = m >= 0 && m < a.n_models;
        const double log_rho = valid ? (double)a.tlogp[r] - (double)a.blogp[r] : 0.0;
        const double rho = exp(log_rho);
        const double rho_c = fmin(rho, a.clip_rho), c = fmin(rho, 1.0), rho_pg = fmin(rho, a.clip_pg_rho);
        const double disc = a.gamma * (1.0 - (a.done[r] ? 1.0 : 0.0));
        const double V = a.value[r], rw = a.reward[r];
        acc = rho_c * (rw + disc * v_next - V) + disc * c * acc;
        const double vs = V + acc;
        a.vs[r] = (float)vs;
        a.pg_adv[r] = (float)(rho_pg * (rw + disc * vs_next - V));
        a.lmodel[r] = valid ? m : -1;
        v_next = V; vs_next = vs;
    }
}

// one SGD step's statistics (RAMP_IMPALA_*): the loss's sums over the loss rows, their mean entropy and rho, the gradient's
// global norm before clipping.  rows of the step: launch row i is batch row row0 + i.
__global__ void ramp_impala_step_stats_kernel(const float* row_stats, const int32_t* row_model, int32_t rows, int32_t row0,
                                              const float* log_rho, double vf_coeff, double ent_coeff, const double* norm_part,
                                              double* out) {
    double pi = 0.0, vf = 0.0, ent = 0.0, rho = 0.0;
    int n = 0;
    for (int i = 0; i < rows; ++i) {
        if (row_model[i] < 0) continue;
        const float* s = row_stats + (size_t)i * RS_N;
        pi += s[RS_PI]; vf += s[RS_VF]; ent += s[RS_ENT];
        rho += exp((double)log_rho[row0 + i]);
        ++n;
    }
    out[RAMP_IMPALA_TOTAL_LOSS] = pi + vf_coeff * vf - ent_coeff * ent;
    out[RAMP_IMPALA_POLICY_LOSS] = pi; out[RAMP_IMPALA_VF_LOSS] = vf;
    out[RAMP_IMPALA_ENTROPY] = n ? ent / n : 0.0; out[RAMP_IMPALA_MEAN_RHO] = n ? rho / n : 0.0;
    out[RAMP_IMPALA_GRAD_NORM] = sum_norm_parts(norm_part); out[RAMP_IMPALA_ROWS] = n; out[RAMP_IMPALA_SGD_STEPS] = 1;
}

// the means over the call's SGD steps, and their number
__global__ void ramp_impala_learn_stats_kernel(const double* step_stats, int32_t n_steps, double* out) {
    for (int j = 0; j < RAMP_IMPALA_STATS_LEN; ++j) {
        double s = 0.0;
        for (int i = 0; i < n_steps; ++i) s += step_stats[(size_t)i * RAMP_IMPALA_STATS_LEN + j];
        out[j] = n_steps ? s / n_steps : 0.0;
    }
    out[RAMP_IMPALA_SGD_STEPS] = n_steps;
}

// ---- PG (ramp_policy_learn_pg, ramp_pg_loss_grad) ----

// PG's statistics (RAMP_PG_*) over the launch's first min(mb, *n_rows) rows (row i is batch row i: PG does not shuffle):
// policy_loss = -sum(logp(a) adv) / rows, the rows the head-gradient kernel divides by; the mean entropy over the rows with a
// decision
__global__ void ramp_pg_stats_kernel(const float* row_stats, const int32_t* row_model, const float* adv, int32_t mb, const int32_t* n_rows,
                                     const double* norm_part, double* out) {
    const int rows = max(0, min(mb, *n_rows));
    double pi = 0.0, ent = 0.0;
    int k = 0;
    for (int i = 0; i < rows; ++i) {
        if (row_model[i] < 0) continue;
        const float* s = row_stats + (size_t)i * RS_N;
        pi += (double)s[RS_PI] * (double)adv[i]; ent += s[RS_ENT];
        ++k;
    }
    out[RAMP_PG_POLICY_LOSS] = rows ? -pi / rows : 0.0;
    out[RAMP_PG_ENTROPY] = k ? ent / k : 0.0;
    out[RAMP_PG_GRAD_NORM] = sum_norm_parts(norm_part);
    out[RAMP_PG_ROWS] = rows;
}

}  // namespace ramp
