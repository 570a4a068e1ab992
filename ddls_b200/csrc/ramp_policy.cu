// ramp_policy.cu -- the GNN policy forward on the device (include/ramp_b200.h: ramp_policy_*; SURVEY.md 8f-3).
//
// Restates GNNPolicy.forward (ml_models/policies/gnn_policy.py:137-296) for the observation RampJobPartitioningEnvironment
// emits.  Two kernels, both fp32:
//
//   ramp_gnn_embed_kernel   one CTA per job type.  num_rounds x MeanPool (ml_models/models/mean_pool.py:107-150): node module
//                           LN -> Linear -> act per node, edge module per edge, then per destination node the mean over
//                           [own (node | zeros) state, incoming (src node | edge) messages] of reduce module LN -> Linear -> act;
//                           a node with no incoming edge ends a round with zeros (DGL update_all).  Then the mean over the nodes
//                           (gnn_policy.py:262-268).  A job type's node / edge features never change (observation.py:503-567), so
//                           this runs once per weight set, not per decision.
//   ramp_policy_head_kernel persistent CTAs, one warp per episode: graph module LN -> Linear over [graph features | action mask]
//                           (gnn_policy.py:96-109, 271), concat with the model's node-mean embedding, the RLlib fully-connected
//                           read-out (one hidden layer, logits; a separate value branch, or under vf_share_layers the value
//                           layer on the policy's hidden layer), + max(log(mask), FLT_MIN) on the logits
//                           (gnn_policy.py:283-290), then greedy / categorical action selection written straight into the
//                           environment's action buffer.  All read-out weights are staged once per CTA in shared memory, laid
//                           out so that lanes read consecutive words.
//
// Each forward's statements exist once: meanpool_round / node_mean / gnn_embed_body for the embedding, head_row for one
// episode's read-out.  The kernels here, ES's (ramp_es.cuh), the learner's forward (ramp_policy_learn.cuh) and the population's
// (ramp_population.cuh) all run them, each with its own weight blob and launch shape, so a weight set gives the same bits in every
// one of them.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <vector>

#include "ramp_owned.cuh"

cudaStream_t ramp_internal_stream(ramp_engine_t* e);
int ramp_internal_device(ramp_engine_t* e);
void ramp_internal_count_launches(ramp_engine_t* e, int n);

namespace ramp {

constexpr int POL_MAX_ROUNDS = 8;
constexpr int POL_MAX_DIM = 128;        // node / message / embedding widths
constexpr int POL_MAX_HPL = 16;         // read-out hidden units per lane (hidden <= 512)
constexpr float LN_EPS = 1e-5f;         // torch.nn.LayerNorm default

struct RoundW {                          // offsets (in floats) into the weight blob
    int32_t in, out;
    int64_t nln_w, nln_b, nW, nb, eln_w, eln_b, eW, eb, rln_w, rln_b, rW, rb;
};

struct PolicyDev {
    ramp_policy_config_t c;
    RoundW rounds[POL_MAX_ROUNDS];
    int64_t gln_w, gln_b, gW, gb, hW, hb, lW, lb, vhW, vhb, vW, vb;
    const float* w;                      // the blob
};

struct ModelDev {
    int32_t n_nodes, n_edges;
    const float* nf; const float* ef;    // [N][in_node], [E][in_edge]
    const int32_t* in_ptr; const int32_t* in_edge; const int32_t* in_src;   // CSR by destination
    float* z0; float* z1;                // [N][POL_MAX_DIM]
    float* hn; float* he;                // [N][msg/2], [E][msg/2]
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ float act_fn(float x, int kind) {
    if (kind == 0) return fmaxf(x, 0.f);
    if (kind == 1) return x > 0.f ? x : 0.01f * x;
    return tanhf(x);
}

// LayerNorm of the n values a warp holds lane-strided in `buf` (shared, per warp), in place: biased variance, eps inside the root
__device__ __forceinline__ void warp_layer_norm(float* buf, int n, const float* w, const float* b, int lane) {
    float s = 0.f;
    for (int k = lane; k < n; k += 32) s += buf[k];
    const float mean = warp_sum(s) / (float)n;
    float q = 0.f;
    for (int k = lane; k < n; k += 32) { const float d = buf[k] - mean; q += d * d; }
    const float rstd = 1.0f / sqrtf(warp_sum(q) / (float)n + LN_EPS);
    for (int k = lane; k < n; k += 32) buf[k] = (buf[k] - mean) * rstd * w[k] + b[k];
    __syncwarp();
}

// One MeanPool round (mean_pool.py:120-150) with the weight blob `w` on M's graph, by the whole CTA: the round's input zin (rows
// zin_stride apart) -> its output zout (rows zout_stride apart); hn / he get the node and edge modules' outputs.  buf: this warp's
// POL_MAX_DIM floats of shared staging.  Every forward of the rounds runs these statements, so they give the same bits.
__device__ __forceinline__ void meanpool_round(const PolicyDev& P, const float* w, const RoundW& R, const ModelDev& M, const float* zin,
                                               int zin_stride, float* zout, int zout_stride, float* hn, float* he, float* buf) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
    const int half = P.c.out_features_msg / 2, msg = P.c.out_features_msg, akind = P.c.aggregator_activation;
    // ---- node module on every node, edge module on every edge (mean_pool.py:120-127) ----
    for (int v = warp; v < M.n_nodes; v += n_warps) {
        for (int k = lane; k < R.in; k += 32) buf[k] = zin[(size_t)v * zin_stride + k];
        __syncwarp();
        warp_layer_norm(buf, R.in, w + R.nln_w, w + R.nln_b, lane);
        for (int o = lane; o < half; o += 32) {
            float a = w[R.nb + o];
            const float* row = w + R.nW + (size_t)o * R.in;
            for (int k = 0; k < R.in; ++k) a += row[k] * buf[k];
            hn[(size_t)v * half + o] = act_fn(a, akind);
        }
        __syncwarp();
    }
    const int ine = P.c.in_features_edge;
    for (int e = warp; e < M.n_edges; e += n_warps) {
        for (int k = lane; k < ine; k += 32) buf[k] = M.ef[(size_t)e * ine + k];
        __syncwarp();
        warp_layer_norm(buf, ine, w + R.eln_w, w + R.eln_b, lane);
        for (int o = lane; o < half; o += 32) {
            float a = w[R.eb + o];
            const float* row = w + R.eW + (size_t)o * ine;
            for (int k = 0; k < ine; ++k) a += row[k] * buf[k];
            he[(size_t)e * half + o] = act_fn(a, akind);
        }
        __syncwarp();
    }
    __syncthreads();
    // ---- per destination node: mean of reduce_module over [own state, messages] (mean_pool.py:129-150) ----
    for (int v = warp; v < M.n_nodes; v += n_warps) {
        const int e0 = M.in_ptr[v], e1 = M.in_ptr[v + 1];
        float acc[POL_MAX_DIM / 32];
#pragma unroll
        for (int i = 0; i < POL_MAX_DIM / 32; ++i) acc[i] = 0.f;
        if (e1 > e0) {                                              // DGL leaves zero-in-degree nodes at zero
            for (int mi = -1; mi < e1 - e0; ++mi) {
                const int src = mi < 0 ? v : M.in_src[e0 + mi];
                for (int k = lane; k < half; k += 32) {
                    buf[k] = hn[(size_t)src * half + k];
                    buf[half + k] = mi < 0 ? 0.f : he[(size_t)M.in_edge[e0 + mi] * half + k];
                }
                __syncwarp();
                warp_layer_norm(buf, msg, w + R.rln_w, w + R.rln_b, lane);
#pragma unroll
                for (int i = 0; i < POL_MAX_DIM / 32; ++i) {
                    const int o = lane + 32 * i;
                    if (o < R.out) {
                        float a = w[R.rb + o];
                        const float* row = w + R.rW + (size_t)o * msg;
                        for (int k = 0; k < msg; ++k) a += row[k] * buf[k];
                        acc[i] += act_fn(a, akind);
                    }
                }
                __syncwarp();
            }
        }
        const float inv = 1.0f / (float)(e1 - e0 + 1);
#pragma unroll
        for (int i = 0; i < POL_MAX_DIM / 32; ++i) {
            const int o = lane + 32 * i;
            if (o < R.out) zout[(size_t)v * zout_stride + o] = acc[i] * inv;
        }
    }
    __syncthreads();
}

// the mean over the job's n_nodes node states (rows `stride` apart) into emb_out[od] (gnn_policy.py:262-268), by the whole CTA.
// The sum runs in double: an fp32 running sum of thousands of like-signed states drifts by ~n ulp (5.6e-5 relative on a 4,097-node
// out-star of single-unit states)
__device__ __forceinline__ void node_mean(const float* z, int stride, int n_nodes, int od, float* emb_out) {
    for (int o = threadIdx.x; o < od; o += blockDim.x) {
        double s = 0.0;
        for (int v = 0; v < n_nodes; ++v) s += (double)z[(size_t)v * stride + o];
        emb_out[o] = (float)(s / (double)n_nodes);
    }
}

// the embedding of one job type with the weight blob `w` into emb_out[out_node], by the whole CTA; M's z0 / z1 (ping-pong round
// states) and hn / he are the scratch
__device__ __forceinline__ void gnn_embed_body(const PolicyDev& P, const float* w, const ModelDev& M, float* emb_out) {
    __shared__ float sbuf[8][POL_MAX_DIM];
    if (M.n_nodes <= 0) return;
    float* buf = sbuf[threadIdx.x >> 5];
    const float* zin = M.nf;
    int zin_stride = P.c.in_features_node;
    float* zout = M.z0;
    for (int r = 0; r < P.c.num_rounds; ++r) {
        const RoundW R = P.rounds[r];
        meanpool_round(P, w, R, M, zin, zin_stride, zout, POL_MAX_DIM, M.hn, M.he, buf);
        zin = zout; zin_stride = POL_MAX_DIM;
        zout = (zout == M.z0) ? M.z1 : M.z0;
    }
    node_mean(zin, POL_MAX_DIM, M.n_nodes, P.c.out_features_node, emb_out);
}

__global__ void __launch_bounds__(256) ramp_gnn_embed_kernel(const PolicyDev P, const ModelDev* models, float* emb) {
    gnn_embed_body(P, P.w, models[blockIdx.x], emb + (size_t)blockIdx.x * P.c.out_features_node);
}

struct HeadArgs {
    int32_t n;                            // decisions
    // inputs: either full graph features (host-style forward) or the environment's buffers
    const float* graph_features;          // [n][in_graph] or nullptr
    const float* obs_dyn;                 // [n][11]
    const float* graph_static;            // [n_models][6]
    const int32_t* model;                 // [n]
    const uint8_t* done;                  // [n] or nullptr
    const uint8_t* mask;                  // [n][A]
    const float* emb;                     // [n_models][out_node]
    float* logits; float* value; float* logp; int32_t* actions;   // outputs (logits / value / logp may be nullptr)
    int32_t sample;
    unsigned long long seed;
};

__host__ __device__ inline size_t head_smem_floats(const ramp_policy_config_t& c, int warps) {
    const int gin = c.in_features_graph + c.n_actions, fin = c.out_features_node + c.out_features_graph, A = c.n_actions;
    const size_t layers = c.vf_share_layers ? 1 : 2, Hp = 32 * (size_t)((c.fcnet_hidden + 31) / 32);
    return (size_t)2 * gin + (size_t)c.out_features_graph * gin + c.out_features_graph      // graph module
           + layers * (fin * Hp + Hp)                                                      // hidden layers (policy, value), transposed
           + (size_t)A * Hp + A + Hp + 1                                                    // logits, value
           + (size_t)warps * 2 * POL_MAX_DIM;                                               // per-warp staging
}

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// The read-out's weights in one of two layouts, read by head_row.  ReadoutStaged: head_body's per-CTA copy in shared memory, the
// hidden and logit weights transposed to [fin][Hp] / [A][Hp] so that lanes read consecutive hidden units, padded with zero
// weights and biases to Hp, a multiple of 32 (Hp = H when 32 | H).  ReadoutBlob: the blob's own [H][fin] / [A][H] rows in global
// memory.  A lane owns the hidden units lane + 32 i, i < units(lane): Hp / 32 of them in the staged copy, padding included -- a
// padding unit is 0 and adds exactly 0 to a split-K sum that starts from +0, so both layouts give the same bits.
struct ReadoutWeights { const float *gln_w, *gln_b, *gW, *gb, *hW, *hb, *vhW, *vhb, *lW, *lb, *vW, *vb; };

struct ReadoutStaged : ReadoutWeights {
    int Hp;
    __device__ int units(int) const { return Hp / 32; }
    __device__ float hw(const float* W, int k, int j) const { return W[(size_t)k * Hp + j]; }     // hidden unit j, input k
    __device__ float lw(int o, int j) const { return lW[(size_t)o * Hp + j]; }                  // logit o, hidden unit j
};

struct ReadoutBlob : ReadoutWeights {
    int H, fin;
    __device__ ReadoutBlob(const PolicyDev& P, const float* w)
        : ReadoutWeights{w + P.gln_w, w + P.gln_b, w + P.gW, w + P.gb, w + P.hW, w + P.hb, w + P.vhW, w + P.vhb, w + P.lW, w + P.lb, w + P.vW, w + P.vb},
          H(P.c.fcnet_hidden), fin(P.c.out_features_node + P.c.out_features_graph) {}
    __device__ int units(int lane) const { return (H - lane + 31) / 32; }
    __device__ float hw(const float* W, int k, int j) const { return W[(size_t)j * fin + k]; }
    __device__ float lw(int o, int j) const { return lW[(size_t)o * H + j]; }
};

// The read-out of episode / row b with the weights W, by one warp (gnn_policy.py:96-109, 262-290): [graph features | action
// mask] -> LN -> Linear, concat with the job type's embedding emb[m], the hidden layer(s), the logits + max(log(mask), FLT_MIN),
// the value (only when a.value is given), then the first maximal logit or a categorical draw.  xb: this warp's 2 POL_MAX_DIM
// floats of shared staging.
template <class W_>
__device__ __forceinline__ void head_row(const ramp_policy_config_t& c, const W_& W, const HeadArgs& a, const float* emb, int b, float* xb,
                                         int lane) {
    const int gin = c.in_features_graph + c.n_actions, og = c.out_features_graph, on = c.out_features_node, fin = on + og;
    const int A = c.n_actions, hpl = W.units(lane);
    const int m = a.model[b];
    const bool live = m >= 0 && m < c.n_models && !(a.done && a.done[b]);
    if (!live) {                                                        // nothing queued: the action is ignored by the environment
        if (lane < A && a.logits) a.logits[(size_t)b * A + lane] = 0.f;
        if (lane == 0) { a.actions[b] = 0; if (a.value) a.value[b] = 0.f; if (a.logp) a.logp[b] = 0.f; }
        return;
    }
    float* fb = xb + POL_MAX_DIM;
    // ---- [graph features | action mask] (observation.py:298-300) -> LN -> Linear (gnn_policy.py:96-109) ----
    for (int k = lane; k < gin; k += 32) {
        float x;
        if (k >= c.in_features_graph) x = a.mask[(size_t)b * A + (k - c.in_features_graph)] ? 1.f : 0.f;
        else if (a.graph_features) x = a.graph_features[(size_t)b * c.in_features_graph + k];
        else if (k < 9) x = a.obs_dyn[(size_t)b * 11 + k];
        else if (k < 15) x = a.graph_static[(size_t)m * 6 + (k - 9)];
        else x = a.obs_dyn[(size_t)b * 11 + (k - 6)];
        xb[k] = x;
    }
    __syncwarp();
    warp_layer_norm(xb, gin, W.gln_w, W.gln_b, lane);
    for (int k = lane; k < on; k += 32) fb[k] = emb[(size_t)m * on + k];
    if (lane < og) {
        float g = W.gb[lane];
        const float* row = W.gW + (size_t)lane * gin;
        for (int k = 0; k < gin; ++k) g += row[k] * xb[k];
        fb[on + lane] = g;
    }
    __syncwarp();
    // ---- read-out: hidden layer of the policy and of the value branch, each lane owns units lane + 32 i ----
    float h[POL_MAX_HPL], hv[POL_MAX_HPL];
    if (c.vf_share_layers || !a.value) {                                // no value hidden layer (the value reads h), or no value
#pragma unroll
        for (int i = 0; i < POL_MAX_HPL; ++i) {
            if (i < hpl) {
                const int j = lane + 32 * i;
                float p = W.hb[j];
                for (int k = 0; k < fin; ++k) p += W.hw(W.hW, k, j) * fb[k];
                h[i] = hv[i] = act_fn(p, c.fcnet_activation);
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < POL_MAX_HPL; ++i) {
            if (i < hpl) {
                const int j = lane + 32 * i;
                float p = W.hb[j], q = W.vhb[j];
                for (int k = 0; k < fin; ++k) { const float f = fb[k]; p += W.hw(W.hW, k, j) * f; q += W.hw(W.vhW, k, j) * f; }
                h[i] = act_fn(p, c.fcnet_activation); hv[i] = act_fn(q, c.fcnet_activation);
            }
        }
    }
    float my_logit = -FLT_MAX;
    for (int o = 0; o < A; ++o) {
        float p = 0.f;
#pragma unroll
        for (int i = 0; i < POL_MAX_HPL; ++i) if (i < hpl) p += h[i] * W.lw(o, lane + 32 * i);
        p = warp_sum(p) + W.lb[o];
        if (c.apply_action_mask && !a.mask[(size_t)b * A + o]) p += -FLT_MAX;   // + max(log 0, finfo.min) (gnn_policy.py:285-290)
        if (lane == o) my_logit = p;
    }
    float val = 0.f;
    if (a.value) {
#pragma unroll
        for (int i = 0; i < POL_MAX_HPL; ++i) if (i < hpl) val += hv[i] * W.vW[lane + 32 * i];
        val = warp_sum(val) + W.vb[0];
    }
    // ---- action: first maximal logit, or a categorical draw over softmax(logits) ----
    float best = my_logit; int arg = lane < A ? lane : 0x7fffffff;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
        if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
    }
    const float ex = lane < A ? expf(my_logit - best) : 0.f;
    const float denom = warp_sum(ex);
    int action = arg;
    if (a.sample) {
        float cum = ex;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const float t = __shfl_up_sync(0xffffffffu, cum, o); if (lane >= o) cum += t; }
        const unsigned long long r = splitmix64(a.seed ^ ((unsigned long long)b * 0xD1342543DE82EF95ull));
        const float u = (float)(r >> 40) * (1.0f / 16777216.0f) * denom;
        const unsigned ok = __ballot_sync(0xffffffffu, lane < A && ex > 0.f && cum > u);
        action = ok ? __ffs(ok) - 1 : arg;
    }
    const float chosen = __shfl_sync(0xffffffffu, my_logit, action);
    if (lane < A && a.logits) a.logits[(size_t)b * A + lane] = my_logit;
    if (lane == 0) {
        a.actions[b] = action;
        if (a.value) a.value[b] = val;
        if (a.logp) a.logp[b] = chosen - best - logf(denom);
    }
    __syncwarp();
}

// ramp_policy_head_kernel's statements with the weight blob `w` (P's layout), CTA `cta` of n_ctas: the read-out weights staged in
// shared memory, then head_row on the CTA's episodes.  Shared with the population's head kernel, which runs one weight set per
// blockIdx.y
__device__ __forceinline__ void head_body(const PolicyDev& P, const float* w, const HeadArgs& a, int cta, int n_ctas) {
    extern __shared__ float sm[];
    const ramp_policy_config_t& c = P.c;
    const int gin = c.in_features_graph + c.n_actions, og = c.out_features_graph, on = c.out_features_node, fin = on + og;
    const int H = c.fcnet_hidden, Hp = 32 * ((H + 31) / 32), A = c.n_actions;
    const bool share = c.vf_share_layers;                             // no value hidden layer
    float* s_gln_w = sm;                 float* s_gln_b = s_gln_w + gin;
    float* s_gW = s_gln_b + gin;         float* s_gb = s_gW + (size_t)og * gin;
    float* s_hWt = s_gb + og;            float* s_hb = s_hWt + (size_t)fin * Hp;     // [fin][Hp]
    float* s_vhWt = s_hb + Hp;           float* s_vhb = s_vhWt + (share ? 0 : (size_t)fin * Hp);
    float* s_lW = s_vhb + (share ? 0 : Hp); float* s_lb = s_lW + (size_t)A * Hp;     // [A][Hp]
    float* s_vW = s_lb + A;              float* s_vb = s_vW + Hp;
    float* s_warp = s_vb + 1;
    for (int i = threadIdx.x; i < gin; i += blockDim.x) { s_gln_w[i] = w[P.gln_w + i]; s_gln_b[i] = w[P.gln_b + i]; }
    for (int i = threadIdx.x; i < og * gin; i += blockDim.x) s_gW[i] = w[P.gW + i];
    for (int i = threadIdx.x; i < og; i += blockDim.x) s_gb[i] = w[P.gb + i];
    for (int i = threadIdx.x; i < fin * H; i += blockDim.x) {
        const int j = i / fin, k = i - j * fin;                       // blob is [H][fin]
        s_hWt[(size_t)k * Hp + j] = w[P.hW + i];
        if (!share) s_vhWt[(size_t)k * Hp + j] = w[P.vhW + i];
    }
    for (int i = threadIdx.x; i < H; i += blockDim.x) { s_hb[i] = w[P.hb + i]; if (!share) s_vhb[i] = w[P.vhb + i]; s_vW[i] = w[P.vW + i]; }
    for (int i = threadIdx.x; i < A * H; i += blockDim.x) { const int o = i / H; s_lW[(size_t)o * Hp + (i - o * H)] = w[P.lW + i]; }
    for (int i = threadIdx.x; i < A; i += blockDim.x) s_lb[i] = w[P.lb + i];
    if (threadIdx.x == 0) s_vb[0] = w[P.vb];
    if (Hp != H) {
        const int pad = Hp - H;
        for (int i = threadIdx.x; i < fin * pad; i += blockDim.x) {
            const int k = i / pad, j = H + (i - k * pad);
            s_hWt[(size_t)k * Hp + j] = 0.f;
            if (!share) s_vhWt[(size_t)k * Hp + j] = 0.f;
        }
        for (int i = threadIdx.x; i < pad; i += blockDim.x) { s_hb[H + i] = 0.f; if (!share) s_vhb[H + i] = 0.f; s_vW[H + i] = 0.f; }
        for (int i = threadIdx.x; i < A * pad; i += blockDim.x) { const int o = i / pad; s_lW[(size_t)o * Hp + H + (i - o * pad)] = 0.f; }
    }
    __syncthreads();

    const ReadoutStaged W{{s_gln_w, s_gln_b, s_gW, s_gb, s_hWt, s_hb, s_vhWt, s_vhb, s_lW, s_lb, s_vW, s_vb}, Hp};
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpc = blockDim.x >> 5;
    float* xb = s_warp + (size_t)warp * 2 * POL_MAX_DIM;                // graph-module input, then the read-out input
    for (int b = cta * wpc + warp; b < a.n; b += n_ctas * wpc) head_row(c, W, a, a.emb, b, xb, lane);
}

// at most 80 registers (three CTAs per SM), what the kernel used before its read-out was padded to Hp: left alone, ptxas takes 113
__global__ void __launch_bounds__(256, 3) ramp_policy_head_kernel(const PolicyDev P, const HeadArgs a) {
    head_body(P, P.w, a, blockIdx.x, gridDim.x);
}

// one launch per phase instead of a handful of small device-to-device copies
struct TrajArgs {
    int32_t B, A, phase;
    const float* obs; const int32_t* model; const uint8_t* mask; const int32_t* action; const float* logp; const float* value;
    const double* reward; const uint8_t* done;
    float* t_obs; int32_t* t_model; uint8_t* t_mask; int32_t* t_action; float* t_logp; float* t_value; double* t_reward; uint8_t* t_done;
};

__global__ void ramp_trajectory_record_kernel(const TrajArgs a) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.B) return;
    if (a.phase == 0) {
        for (int k = 0; k < 11; ++k) a.t_obs[(size_t)b * 11 + k] = a.obs[(size_t)b * 11 + k];
        for (int k = 0; k < a.A; ++k) a.t_mask[(size_t)b * a.A + k] = a.mask[(size_t)b * a.A + k];
        a.t_model[b] = a.model[b]; a.t_action[b] = a.action[b]; a.t_logp[b] = a.logp[b]; a.t_value[b] = a.value[b];
    } else {
        a.t_reward[b] = a.reward[b]; a.t_done[b] = a.done[b];
    }
}

// ramp_policy_forward_device / ramp_policy_backward_device: caller-owned device rows gathered into the staging buffers the host
// paths upload into, so that every kernel after this one runs on its usual inputs
struct PolicyIngestArgs {
    int32_t n, is64, n_models, in_graph, A;
    int64_t gf_stride;                    // floats from one graph_features row to the next (>= in_graph)
    const void* model; const float* graph_features; const uint8_t* mask; const float* grad_logits; const float* grad_value;
    int32_t* model_out; float* gf_out; uint8_t* mask_out;
    float* gl_out; float* gv_out;         // nullptr: a forward
    int32_t* n_rows_out;                  // the row count for the gradient kernels, or nullptr
};

// one thread per (row, column): column k < in_graph gathers a graph feature, k < A a mask byte (and a logit's upstream
// gradient); column 0 the model, as int32 -- any value outside [0, n_models) becomes -1, so an int64 is never wrapped into range
__global__ void ramp_policy_ingest_kernel(const PolicyIngestArgs a) {
    const int W = a.in_graph > a.A ? a.in_graph : a.A;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)a.n * W) return;
    const int b = (int)(i / W), k = (int)(i - (long long)b * W);
    if (k < a.in_graph) a.gf_out[(size_t)b * a.in_graph + k] = a.graph_features[(size_t)b * a.gf_stride + k];
    if (k < a.A) {
        const size_t o = (size_t)b * a.A + k;
        a.mask_out[o] = a.mask[o] ? 1 : 0;
        if (a.gl_out) a.gl_out[o] = a.grad_logits[o];
    }
    if (k == 0) {
        const long long x = a.is64 ? static_cast<const long long*>(a.model)[b] : (long long)static_cast<const int32_t*>(a.model)[b];
        a.model_out[b] = x >= 0 && x < a.n_models ? (int32_t)x : -1;
        if (a.gv_out) a.gv_out[b] = a.grad_value[b];
        if (b == 0 && a.n_rows_out) *a.n_rows_out = a.n;
    }
}

}  // namespace ramp

#include "ramp_policy_learn.cuh"

using namespace ramp;

struct HostModel {
    ModelDev d{};
    std::vector<DeviceArray<unsigned char>> allocs;
    bool set = false;
    GradModelDev g{};                     // the out-edge CSR (with `allocs`) and the learner's scratch (`lallocs`, made on first use)
    std::vector<DeviceArray<unsigned char>> lallocs;
    bool grad_ready = false;
};

struct SegTable { DeviceArray<Seg> d; int32_t count = 0; int64_t total = 0; };

// The learner's device buffers for K weight sets, stacked set-major: the single policy holds them with K = 1, a population
// (ramp_population.cuh) with its K.  Each capacity stays 0 until every buffer it covers has the new size.
struct LearnerBuffers {
    int32_t K = 1;
    // gradient, Adam's moments and step counts (two per set, read and written by alternate steps: `parity`), per job type
    // gradients, norm partials, statistics, each minibatch's statistics, the train batch's row count per set
    bool ready = false;
    int32_t parity = 0;
    DeviceArray<float> grad, adam_m, adam_v, gpart;
    DeviceArray<int32_t> step, n_rows;
    DeviceArray<double> norm_part, stats, mb_stats;
    // every (set, job type)'s MeanPool states and backward scratch, [K][n_models]
    bool gmodels_ready = false;
    DeviceArray<GradModelDev> gmodels;
    // per-row scratch for K minibatches of `lcap` rows; the head segments of set 0's records for every row count seen since `rec`
    // was last allocated (a segment points into rec), `segs` those of the current one
    int32_t lcap = 0;
    DeviceArray<float> rec, row_stats;
    DeviceArray<int32_t> row_model;
    std::map<int32_t, SegTable> seg_tables;
    const SegTable* segs = nullptr;
    // the train batch (K groups of [horizon * b] rows, live rows first, t-major) and the bootstrap values ([B])
    int32_t bcap = 0, boot_cap = 0;
    DeviceArray<float> b_obs, b_logp, b_logp_old, b_adv, b_vt, b_old, b_value, b_lpx, boot;
    DeviceArray<int32_t> b_model, b_action, b_actx, boot_act; DeviceArray<uint8_t> b_mask; DeviceArray<double> b_adv64;
    // IMPALA (ramp_policy_learn_impala / ramp_impala_loss_grad / ramp_population_learn_impala): K groups of fragment rows ([icap]
    // each, set s's i_rows rows at s i_rows, row f L + t) with their read-out at the current weights and V-trace values, the loss's
    // job types (-1 outside it), the host batch's extra inputs; per set the row count, the statistics and each SGD step's
    int32_t icap = 0, i_rows = 0, i_step_cap = 0;
    DeviceArray<float> i_obs, i_blogp, i_tlogits, i_tvalue, i_tlogp, i_log_rho, i_vs, i_pg;
    DeviceArray<int32_t> i_model, i_action, i_actx, i_lmodel, i_n_rows; DeviceArray<uint8_t> i_mask, i_done;
    DeviceArray<double> i_reward, i_step_stats, i_stats;
};

struct ramp_policy {
    int device = 0;
    PolicyDev P{};
    int64_t n_weights = 0;
    DeviceArray<float> d_w;
    std::vector<HostModel> models;
    DeviceArray<ModelDev> d_models;
    DeviceArray<float> d_emb;             // [n_models][out_node]
    DeviceArray<float> d_gstatic;         // [n_models][6]
    bool weights_set = false, emb_valid = false;
    int sm_count = 132;
    size_t head_smem = 0;
    // outputs of the last act, for ramp_policy_read and ramp_policy_trajectory_record; act_n: its environment's episodes (-1: none yet)
    int32_t cap = 0, act_n = -1;
    DeviceArray<float> d_logits, d_value, d_logp;
    // inputs and outputs of ramp_policy_forward / ramp_policy_decide, apart from act's
    int32_t fcap = 0;
    DeviceArray<int32_t> f_model, f_actions; DeviceArray<float> f_gf, f_logits, f_value, f_logp; DeviceArray<uint8_t> f_mask;
    // a forward captured into a CUDA graph (ramp_policy_forward_device) holds the f_* addresses for the graph's life, which the
    // policy cannot see end: once one was captured, staging that grows is kept here until the policy is destroyed, not freed
    bool fwd_captured = false;
    std::vector<DeviceArray<int32_t>> kept_i32; std::vector<DeviceArray<float>> kept_f32; std::vector<DeviceArray<uint8_t>> kept_u8;
    unsigned long long act_calls = 0;
    // trajectory of a rollout segment (ramp_policy_trajectory_*): [horizon][B] per field, on the device until read
    int32_t traj_h = 0, traj_b = 0, traj_a = 0;
    int32_t traj_n = 0;                   // slots recorded in order, both phases, since ramp_policy_trajectory_begin
    DeviceArray<float> t_obs, t_logp, t_value; DeviceArray<int32_t> t_model, t_action;
    DeviceArray<uint8_t> t_mask, t_done; DeviceArray<double> t_reward;
    // learner (ramp_policy_backward / ramp_ppo_loss_grad / ramp_policy_learn / _learn_pg / _learn_impala)
    // states_current: the MeanPool states kept in L.gmodels are those of a whole-batch forward at the current weights
    LearnerBuffers L;
    bool states_current = false;
    // the end of the last call that touched the scratch above, the staging or the embeddings (made by the first device-path call;
    // until then every call keeps its own synchronisation and nothing is recorded)
    Event ev_done;
    // host-input batches of ramp_policy_backward / ramp_ppo_loss_grad, and their row count on the device
    int32_t hcap = 0;
    DeviceArray<int32_t> h_model, h_action, h_n_rows; DeviceArray<float> h_gf, h_gl, h_gv, h_old, h_adv, h_vt; DeviceArray<uint8_t> h_mask;
    int32_t b_rows = 0;                   // the rows of the last train batch (ramp_policy_train_batch_read)
};

namespace {

int64_t layout(const ramp_policy_config_t& c, PolicyDev* P) {
    int64_t o = 0;
    auto take = [&](int64_t n) { const int64_t at = o; o += n; return at; };
    const int half = c.out_features_msg / 2;
    for (int r = 0; r < c.num_rounds; ++r) {
        const int in = r == 0 ? c.in_features_node : c.out_features_hidden;
        const int out = r == c.num_rounds - 1 ? c.out_features_node : c.out_features_hidden;
        RoundW R{};
        R.in = in; R.out = out;
        R.nln_w = take(in); R.nln_b = take(in); R.nW = take((int64_t)half * in); R.nb = take(half);
        R.eln_w = take(c.in_features_edge); R.eln_b = take(c.in_features_edge); R.eW = take((int64_t)half * c.in_features_edge); R.eb = take(half);
        R.rln_w = take(c.out_features_msg); R.rln_b = take(c.out_features_msg); R.rW = take((int64_t)out * c.out_features_msg); R.rb = take(out);
        if (P) P->rounds[r] = R;
    }
    const int gin = c.in_features_graph + c.n_actions, fin = c.out_features_node + c.out_features_graph, H = c.fcnet_hidden;
    const int64_t gln_w = take(gin), gln_b = take(gin), gW = take((int64_t)c.out_features_graph * gin), gb = take(c.out_features_graph);
    const int64_t hW = take((int64_t)H * fin), hb = take(H), lW = take((int64_t)c.n_actions * H), lb = take(c.n_actions);
    const int64_t vhW = c.vf_share_layers ? -1 : take((int64_t)H * fin), vhb = c.vf_share_layers ? -1 : take(H);   // no value hidden layer
    const int64_t vW = take(H), vb = take(1);
    if (P) { P->gln_w = gln_w; P->gln_b = gln_b; P->gW = gW; P->gb = gb; P->hW = hW; P->hb = hb; P->lW = lW; P->lb = lb;
             P->vhW = vhW; P->vhb = vhb; P->vW = vW; P->vb = vb; }
    return o;
}

int check_config(const ramp_policy_config_t& c) {
    auto in = [](int v, int lo, int hi) { return v >= lo && v <= hi; };
    if (!in(c.in_features_node, 1, POL_MAX_DIM) || !in(c.in_features_edge, 1, POL_MAX_DIM) || !in(c.in_features_graph, 1, POL_MAX_DIM - 32))
        return set_error(RAMP_ERR_BAD_ARG, "policy: feature widths must be in [1, %d]", POL_MAX_DIM);
    if (!in(c.out_features_msg, 2, POL_MAX_DIM) || (c.out_features_msg & 1) || !in(c.out_features_hidden, 1, POL_MAX_DIM) || !in(c.out_features_node, 1, POL_MAX_DIM - 32))
        return set_error(RAMP_ERR_BAD_ARG, "policy: out_features_msg must be even and every width <= %d", POL_MAX_DIM);
    if (!in(c.out_features_graph, 1, 32) || !in(c.n_actions, 1, 32) || c.in_features_graph + c.n_actions > POL_MAX_DIM)
        return set_error(RAMP_ERR_BAD_ARG, "policy: out_features_graph and n_actions must be <= 32");
    if (c.num_rounds < 2 || c.num_rounds > POL_MAX_ROUNDS) return set_error(RAMP_ERR_BAD_ARG, "policy: num_rounds must be in [2, %d] (gnn.py:40-41)", POL_MAX_ROUNDS);
    // a multiple of 32, or action_space.n: the width the algorithm configs set (algo/{ppo,impala,pg,es}.yaml), at most 32
    const bool h32 = c.fcnet_hidden >= 32 && c.fcnet_hidden % 32 == 0 && c.fcnet_hidden <= 32 * POL_MAX_HPL;
    if (!h32 && c.fcnet_hidden != c.n_actions)
        return set_error(RAMP_ERR_BAD_ARG, "policy: fcnet_hidden must be a multiple of 32 in [32, %d] or n_actions (%d)", 32 * POL_MAX_HPL, c.n_actions);
    if (!in(c.vf_share_layers, 0, 1)) return set_error(RAMP_ERR_BAD_ARG, "policy: vf_share_layers must be 0 or 1");
    if (!in(c.aggregator_activation, 0, 1) || !(c.fcnet_activation == 0 || c.fcnet_activation == 2))
        return set_error(RAMP_ERR_BAD_ARG, "policy: unsupported activation");
    if (c.n_models < 1) return set_error(RAMP_ERR_BAD_ARG, "policy: n_models must be >= 1");
    return RAMP_OK;
}

int ensure_outputs(ramp_policy* p, int32_t n) {
    if (n <= p->cap) return RAMP_OK;
    p->cap = 0;                           // until every buffer has the new size
    CUDA_TRY(p->d_logits.alloc((size_t)n * p->P.c.n_actions));
    CUDA_TRY(alloc_each(n, p->d_value, p->d_logp));
    p->cap = n;
    return RAMP_OK;
}

// the job-type table d_models is uploaded by ramp_policy_set_model, once per change
int launch_embed(ramp_policy* p, cudaStream_t st) {
    for (size_t m = 0; m < p->models.size(); ++m)
        if (!p->models[m].set) return set_error(RAMP_ERR_BAD_ARG, "policy: model %zu was never registered (ramp_policy_set_model)", m);
    if (!p->weights_set) return set_error(RAMP_ERR_BAD_ARG, "policy: no weights (ramp_policy_set_weights)");
    ramp_gnn_embed_kernel<<<(unsigned)p->models.size(), 256, 0, st>>>(p->P, p->d_models.get(), p->d_emb.get());
    CUDA_TRY(cudaGetLastError());
    p->emb_valid = true;
    p->states_current = false;
    return RAMP_OK;
}

// the policy's scratch is reused by every call: a call's stream first waits for the end of the previous call, on whatever stream
// it ran, and the call then marks its own end.  Both are no-ops until a device-path call made the event.
int fence_in(ramp_policy* p, cudaStream_t st) {
    if (p->ev_done) CUDA_TRY(cudaStreamWaitEvent(st, p->ev_done.get(), 0));
    return RAMP_OK;
}

int fence_out(ramp_policy* p, cudaStream_t st) {
    if (p->ev_done) CUDA_TRY(cudaEventRecord(p->ev_done.get(), st));
    return RAMP_OK;
}

// the f_* staging of the read-out on n rows (ramp_policy_forward / _decide / _forward_device)
int stage_forward(ramp_policy* p, int32_t n) {
    if (n <= p->fcap) return RAMP_OK;
    const ramp_policy_config_t& c = p->P.c;
    p->fcap = 0;                          // until every buffer has the new size
    if (p->fwd_captured) {
        for (DeviceArray<int32_t>* a : {&p->f_model, &p->f_actions}) p->kept_i32.push_back(std::move(*a));
        for (DeviceArray<float>* a : {&p->f_gf, &p->f_logits, &p->f_value, &p->f_logp}) p->kept_f32.push_back(std::move(*a));
        p->kept_u8.push_back(std::move(p->f_mask));
    }
    CUDA_TRY(alloc_each(n, p->f_model, p->f_actions, p->f_value, p->f_logp));
    CUDA_TRY(p->f_gf.alloc((size_t)n * c.in_features_graph));
    CUDA_TRY(alloc_each((size_t)n * c.n_actions, p->f_mask, p->f_logits));
    p->fcap = n;
    return RAMP_OK;
}

int launch_head(ramp_policy* p, const HeadArgs& a, cudaStream_t st) {
    const int wpc = 8;
    int grid = (a.n + wpc - 1) / wpc;
    if (grid > p->sm_count * 2) grid = p->sm_count * 2;
    if (grid < 1) grid = 1;
    ramp_policy_head_kernel<<<grid, wpc * 32, p->head_smem, st>>>(p->P, a);
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

// the read-out of the n rows staged in f_* on `st`, embedding first when the embeddings are stale; logits / value / logp may be
// nullptr
int launch_forward(ramp_policy* p, cudaStream_t st, int32_t n, int32_t sample, uint64_t seed, float* logits, float* value, float* logp) {
    int rc;
    if (!p->emb_valid && (rc = launch_embed(p, st)) != RAMP_OK) return rc;
    HeadArgs a{};
    a.n = n; a.graph_features = p->f_gf.get(); a.model = p->f_model.get(); a.mask = p->f_mask.get(); a.emb = p->d_emb.get(); a.graph_static = p->d_gstatic.get();
    a.logits = logits; a.value = value; a.logp = logp; a.actions = p->f_actions.get();
    a.sample = sample; a.seed = seed;
    return launch_head(p, a, st);
}

// the read-out on host inputs (ramp_policy_forward / ramp_policy_decide), in buffers of its own: what the last act left for
// ramp_policy_read and the trajectory stays as it was
int head_on_host(ramp_policy* p, int32_t n, const int32_t* model, const float* graph_features, const uint8_t* action_mask, int32_t sample,
                 uint64_t seed, float* logits_out, float* value_out, float* logp_out, int32_t* actions_out) {
    if (!p || !model || !graph_features || !action_mask) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n < 1) return RAMP_OK;
    const ramp_policy_config_t& c = p->P.c;
    CUDA_TRY(cudaSetDevice(p->device));
    int rc;
    if ((rc = fence_in(p, 0)) != RAMP_OK || (rc = stage_forward(p, n)) != RAMP_OK) return rc;
    CUDA_TRY(cudaMemcpy(p->f_model.get(), model, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(p->f_gf.get(), graph_features, sizeof(float) * (size_t)n * c.in_features_graph, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(p->f_mask.get(), action_mask, (size_t)n * c.n_actions, cudaMemcpyHostToDevice));
    if ((rc = launch_forward(p, 0, n, sample, seed, p->f_logits.get(), p->f_value.get(), p->f_logp.get())) != RAMP_OK) return rc;
    CUDA_TRY(cudaStreamSynchronize(0));
    if (logits_out) CUDA_TRY(cudaMemcpy(logits_out, p->f_logits.get(), sizeof(float) * (size_t)n * c.n_actions, cudaMemcpyDeviceToHost));
    if (value_out) CUDA_TRY(cudaMemcpy(value_out, p->f_value.get(), sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
    if (logp_out) CUDA_TRY(cudaMemcpy(logp_out, p->f_logp.get(), sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
    if (actions_out) CUDA_TRY(cudaMemcpy(actions_out, p->f_actions.get(), sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

// ---- the learner ----

uint64_t mix64(uint64_t x) {              // splitmix64, as the kernels' splitmix64
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

int64_t gnn_weight_count(const ramp_policy* p) { return p->P.gln_w; }     // the rounds come first in the blob

// L's gradient, Adam state (zeroed), job-type partials, norm partials and statistics for K sets: n weights and n_gpart job-type
// partials in all
int ensure_learner(LearnerBuffers& L, size_t n, size_t n_gpart) {
    if (L.ready) return RAMP_OK;
    const size_t K = L.K;
    CUDA_TRY(alloc_each(n, L.grad, L.adam_m, L.adam_v));
    CUDA_TRY(L.gpart.alloc(n_gpart));
    CUDA_TRY(L.n_rows.alloc(K));
    CUDA_TRY(L.step.alloc(2 * K));
    CUDA_TRY(L.norm_part.alloc(K * LRN_GRID));
    CUDA_TRY(L.stats.alloc(K * RAMP_PPO_STATS_LEN));
    CUDA_TRY(cudaMemset(L.adam_m.get(), 0, sizeof(float) * n));
    CUDA_TRY(cudaMemset(L.adam_v.get(), 0, sizeof(float) * n));
    CUDA_TRY(cudaMemset(L.step.get(), 0, sizeof(int32_t) * 2 * K));
    L.parity = 0;
    L.ready = true;
    return RAMP_OK;
}

// one job type's forward states and records for the embedding backward (N nodes, E edges), appended to `allocs`
int alloc_grad_scratch(const ramp_policy_config_t& c, size_t N, size_t E, std::vector<DeviceArray<unsigned char>>& allocs, GradModelDev& g) {
    const GnnDims D = gnn_dims(c);
    const size_t half = c.out_features_msg / 2, R = c.num_rounds;
    auto take = [&](size_t floats, float** dst) -> int {
        allocs.emplace_back();
        CUDA_TRY(allocs.back().alloc(sizeof(float) * floats));
        *dst = (float*)allocs.back().get();
        return RAMP_OK;
    };
    int rc;
    if ((rc = take(R * N * D.zs, &g.z)) || (rc = take(R * N * half, &g.hn)) || (rc = take(R * E * half, &g.he)) ||
        (rc = take(N * D.zs, &g.dz)) || (rc = take(N * D.zs, &g.dz2)) || (rc = take(N * half, &g.dhn)) ||
        (rc = take(N * D.nrs, &g.nrec)) || (rc = take(E * D.ers, &g.erec)) || (rc = take((N + E) * D.mrs, &g.mrec)) ||
        (rc = take((N + E) * c.out_features_msg, &g.mdx)))
        return rc;
    return RAMP_OK;
}

// the [K][n_models] table of forward states and backward scratch `h` into L.gmodels, on `st`
int upload_gmodels(LearnerBuffers& L, const std::vector<GradModelDev>& h, cudaStream_t st) {
    if (L.gmodels.size() < h.size()) CUDA_TRY(L.gmodels.alloc(h.size()));
    CUDA_TRY(cudaMemcpyAsync(L.gmodels.get(), h.data(), sizeof(GradModelDev) * h.size(), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));                                  // `h` is pageable
    L.gmodels_ready = true;
    return RAMP_OK;
}

// every job type's forward states and records for the embedding backward, sized by its graph and kept with it
int ensure_gmodels(ramp_policy* p, cudaStream_t st) {
    if (p->L.gmodels_ready) return RAMP_OK;
    std::vector<GradModelDev> h(p->models.size());
    for (size_t m = 0; m < h.size(); ++m) {
        HostModel& hm = p->models[m];
        if (!hm.set) return set_error(RAMP_ERR_BAD_ARG, "policy: model %zu was never registered (ramp_policy_set_model)", m);
        if (!hm.grad_ready) {
            hm.lallocs.clear();
            const int rc = alloc_grad_scratch(p->P.c, hm.d.n_nodes, hm.d.n_edges, hm.lallocs, hm.g);
            if (rc != RAMP_OK) return rc;
            hm.grad_ready = true;
        }
        h[m] = hm.g;
    }
    return upload_gmodels(p->L, h, st);
}

// per-row scratch for K minibatches of n rows, and the head segments summing exactly n of set 0's rows: uploaded on `st` the first
// time n is seen, so a PPO loop whose last minibatch is short does not synchronise every time the row count alternates
int ensure_rows(LearnerBuffers& L, const PolicyDev& P, int32_t n, cudaStream_t st) {
    if (n > L.lcap) {
        const size_t rows = (size_t)L.K * n;
        L.lcap = 0;
        L.segs = nullptr;
        L.seg_tables.clear();
        CUDA_TRY(L.rec.alloc(rows * head_rec(P.c).stride));
        CUDA_TRY(L.row_stats.alloc(rows * RS_N));
        CUDA_TRY(L.row_model.alloc(rows));
        L.lcap = n;
    }
    auto it = L.seg_tables.find(n);
    if (it == L.seg_tables.end()) {
        Seg s[HEAD_SEGS];
        SegTable t;
        t.count = head_segs(P, L.rec.get(), n, s);
        for (int k = 0; k < t.count; ++k) t.total += seg_size(s[k]);
        CUDA_TRY(t.d.alloc(HEAD_SEGS));
        CUDA_TRY(cudaMemcpyAsync(t.d.get(), s, sizeof(s), cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaStreamSynchronize(st));                              // `s` is pageable
        it = L.seg_tables.emplace(n, std::move(t)).first;
    }
    L.segs = &it->second;
    return RAMP_OK;
}

// the train batch for K groups of `rows` trajectory slots each
int ensure_batch(LearnerBuffers& L, const ramp_policy_config_t& c, int32_t rows) {
    if (rows <= L.bcap) return RAMP_OK;
    const size_t n = (size_t)L.K * rows;
    L.bcap = 0;
    CUDA_TRY(alloc_each(n, L.b_logp, L.b_logp_old, L.b_adv, L.b_vt, L.b_value, L.b_lpx, L.b_model, L.b_action, L.b_actx, L.b_adv64));
    CUDA_TRY(L.b_obs.alloc(n * 11));
    CUDA_TRY(alloc_each(n * c.n_actions, L.b_mask, L.b_old));
    L.bcap = rows;
    return RAMP_OK;
}

// a PPO learn call's bootstrap values for B episodes and statistics for K sets of n_mb minibatches
int ensure_ppo(LearnerBuffers& L, int32_t B, int32_t n_mb) {
    if (B > L.boot_cap) {
        L.boot_cap = 0;
        CUDA_TRY(alloc_each(B, L.boot, L.boot_act));
        L.boot_cap = B;
    }
    const size_t n = (size_t)L.K * n_mb * RAMP_PPO_STATS_LEN;
    if (n > L.mb_stats.size()) CUDA_TRY(L.mb_stats.alloc(n));
    return RAMP_OK;
}

// the start of every gradient call on `st`, after the previous call: the learner, every job type's states, current embeddings
// and per-row scratch for minibatches of `rows` rows
int prepare_learner(ramp_policy* p, cudaStream_t st, int32_t rows) {
    int rc;
    if ((rc = fence_in(p, st)) != RAMP_OK || (rc = ensure_learner(p->L, p->n_weights, (size_t)p->P.c.n_models * gnn_weight_count(p))) != RAMP_OK ||
        (rc = ensure_gmodels(p, st)) != RAMP_OK)
        return rc;
    if (!p->emb_valid && (rc = launch_embed(p, st)) != RAMP_OK) return rc;
    return ensure_rows(p->L, p->P, rows, st);
}

// the MeanPool rounds of every job type, kept for the backward (and the embeddings when `emb` is given); nothing for a minibatch
// starting at `start` past the end of a batch of *n_rows rows (n_rows may be nullptr)
int launch_states(ramp_policy* p, cudaStream_t st, const int32_t* n_rows, int32_t start, float* emb) {
    EmbGradArgs eg{};
    eg.n_rows = n_rows; eg.start = start; eg.emb = emb;
    ramp_gnn_embed_grad_kernel<EMB_FORWARD><<<p->P.c.n_models, 256, 0, st>>>(p->P, p->d_models.get(), p->L.gmodels.get(), eg);
    CUDA_TRY(cudaGetLastError());
    p->states_current = n_rows == nullptr;                         // a learn call's minibatch past the batch's end keeps none
    return RAMP_OK;
}

// head gradient -> head reduction -> embedding gradient (from launch_states' states) -> per-job-type sum and norm partials:
// the gradient in l_grad
int launch_grad(ramp_policy* p, GradArgs ga, cudaStream_t st) {
    ga.rec = p->L.rec.get(); ga.row_model = p->L.row_model.get(); ga.row_stats = p->L.row_stats.get();
    ga.emb = p->d_emb.get(); ga.graph_static = p->d_gstatic.get();
    ramp_policy_head_grad_kernel<<<(ga.mb + LRN_WARPS - 1) / LRN_WARPS, LRN_WARPS * 32, 0, st>>>(p->P, ga);
    int64_t grid = (p->L.segs->total + 255) / 256;
    if (grid > 4 * p->sm_count) grid = 4 * p->sm_count;
    ramp_policy_head_reduce_kernel<<<(unsigned)grid, 256, 0, st>>>(p->P, p->L.segs->d.get(), p->L.segs->count, p->L.segs->total, p->L.grad.get());
    EmbGradArgs eg{};
    eg.rec = p->L.rec.get(); eg.row_model = p->L.row_model.get(); eg.rows = ga.mb; eg.gpart = p->L.gpart.get(); eg.n_gnn = gnn_weight_count(p);
    ramp_gnn_embed_grad_kernel<EMB_BACKWARD><<<p->P.c.n_models, 256, 0, st>>>(p->P, p->d_models.get(), p->L.gmodels.get(), eg);
    ramp_grad_finish_kernel<<<LRN_GRID, 256, 0, st>>>(p->L.gpart.get(), p->P.c.n_models, gnn_weight_count(p), p->n_weights,
                                                       p->L.grad.get(), p->L.norm_part.get());
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

int check_learner_config(const ramp_ppo_config_t* cfg) {
    if (!cfg) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (cfg->sgd_minibatch_size < 1 || cfg->num_sgd_iter < 0) return set_error(RAMP_ERR_BAD_ARG, "ppo: sgd_minibatch_size must be >= 1, num_sgd_iter >= 0");
    if (!(cfg->clip_param > 0) || !(cfg->vf_clip_param > 0) || !(cfg->lr >= 0) || !(cfg->adam_eps > 0))
        return set_error(RAMP_ERR_BAD_ARG, "ppo: clip_param, vf_clip_param and adam_eps must be > 0, lr >= 0");
    return RAMP_OK;
}

void ppo_terms(GradArgs& ga, const ramp_ppo_config_t& cfg) {
    ga.clip = (float)cfg.clip_param; ga.vf_clip = (float)cfg.vf_clip_param; ga.vf_coeff = (float)cfg.vf_loss_coeff;
    ga.ent_coeff = (float)cfg.entropy_coeff; ga.kl_coeff = (float)cfg.kl_coeff;
}

// the h_* staging of a batch of n rows (ramp_policy_backward / the loss calls / ramp_policy_backward_device)
int stage_host_batch(ramp_policy* p, int32_t n) {
    if (n <= p->hcap) return RAMP_OK;
    const ramp_policy_config_t& c = p->P.c;
    p->hcap = 0;
    CUDA_TRY(alloc_each(n, p->h_model, p->h_action, p->h_gv, p->h_adv, p->h_vt));
    if (!p->h_n_rows.get()) CUDA_TRY(p->h_n_rows.alloc(1));
    CUDA_TRY(p->h_gf.alloc((size_t)n * c.in_features_graph));
    CUDA_TRY(alloc_each((size_t)n * (size_t)c.n_actions, p->h_gl, p->h_old, p->h_mask));
    p->hcap = n;
    return RAMP_OK;
}

// the host inputs of ramp_policy_backward / ramp_ppo_loss_grad on the device (any pointer may be NULL: not copied)
int upload_host_batch(ramp_policy* p, int32_t n, const int32_t* model, const float* gf, const uint8_t* mask, const float* gl,
                      const float* gv, const int32_t* action, const float* old_logits, const float* adv, const float* vt) {
    const ramp_policy_config_t& c = p->P.c;
    const size_t A = c.n_actions;
    int rc = stage_host_batch(p, n);
    if (rc != RAMP_OK) return rc;
    auto put = [&](void* dst, const void* src, size_t bytes) -> int {
        if (src) CUDA_TRY(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
        return RAMP_OK;
    };
    if ((rc = put(p->h_model.get(), model, 4 * (size_t)n)) || (rc = put(p->h_gf.get(), gf, 4 * (size_t)n * c.in_features_graph)) ||
        (rc = put(p->h_mask.get(), mask, (size_t)n * A)) || (rc = put(p->h_gl.get(), gl, 4 * (size_t)n * A)) ||
        (rc = put(p->h_gv.get(), gv, 4 * (size_t)n)) || (rc = put(p->h_action.get(), action, 4 * (size_t)n)) ||
        (rc = put(p->h_old.get(), old_logits, 4 * (size_t)n * A)) || (rc = put(p->h_adv.get(), adv, 4 * (size_t)n)) ||
        (rc = put(p->h_vt.get(), vt, 4 * (size_t)n)) || (rc = put(p->h_n_rows.get(), &n, 4)))
        return rc;
    for (int32_t b = 0; b < n; ++b)
        if (action && model[b] >= 0 && model[b] < c.n_models && (action[b] < 0 || action[b] >= c.n_actions))
            return set_error(RAMP_ERR_BAD_ARG, "ppo: action %d of row %d outside [0, %d)", action[b], b, c.n_actions);
    return RAMP_OK;
}

GradArgs host_batch_args(ramp_policy* p, int32_t n) {
    GradArgs ga{};
    ga.mb = n; ga.start = 0; ga.n_rows = p->h_n_rows.get();
    ga.graph_features = p->h_gf.get(); ga.model = p->h_model.get(); ga.mask = p->h_mask.get();
    return ga;
}

// the gradient of the n rows staged in h_* (with their upstream gradients h_gl, h_gv) into l_grad, on `st`; the MeanPool states
// are run again unless `reuse_states` and the kept ones are those of the current weights
int launch_backward(ramp_policy* p, cudaStream_t st, int32_t n, bool reuse_states) {
    GradArgs ga = host_batch_args(p, n);
    ga.grad_logits = p->h_gl.get(); ga.grad_value = p->h_gv.get();
    int rc;
    if (!(reuse_states && p->emb_valid && p->states_current) && (rc = launch_states(p, st, nullptr, 0, nullptr)) != RAMP_OK) return rc;
    return launch_grad(p, ga, st);
}

// the caller's device rows into the staging on `st` (ramp_policy_forward_device / _backward_device): model, graph features,
// mask into f_* (gl == nullptr) or h_* with the upstream gradients and the row count
int launch_ingest(ramp_policy* p, cudaStream_t st, int32_t n, const void* model, int32_t model_dtype, const float* graph_features,
                  int64_t gf_stride, const uint8_t* mask, const float* gl, const float* gv) {
    const ramp_policy_config_t& c = p->P.c;
    PolicyIngestArgs a{};
    a.n = n; a.is64 = model_dtype == RAMP_MODEL_INT64; a.n_models = c.n_models; a.in_graph = c.in_features_graph; a.A = c.n_actions;
    a.gf_stride = gf_stride; a.model = model; a.graph_features = graph_features; a.mask = mask; a.grad_logits = gl; a.grad_value = gv;
    if (gl) {
        a.model_out = p->h_model.get(); a.gf_out = p->h_gf.get(); a.mask_out = p->h_mask.get();
        a.gl_out = p->h_gl.get(); a.gv_out = p->h_gv.get(); a.n_rows_out = p->h_n_rows.get();
    } else {
        a.model_out = p->f_model.get(); a.gf_out = p->f_gf.get(); a.mask_out = p->f_mask.get();
    }
    const long long threads = (long long)n * std::max(c.in_features_graph, c.n_actions);
    ramp_policy_ingest_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(a);
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

// the checks every device-path call makes; creates the fencing event on the first one
int device_call_ready(ramp_policy* p, int32_t n, const void* model, int32_t model_dtype, const float* graph_features, int64_t gf_stride,
                      const uint8_t* mask) {
    if (!model || !graph_features || !mask) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (model_dtype != RAMP_MODEL_INT32 && model_dtype != RAMP_MODEL_INT64)
        return set_error(RAMP_ERR_BAD_ARG, "policy: model dtype %d is neither RAMP_MODEL_INT32 nor RAMP_MODEL_INT64", model_dtype);
    if (gf_stride < p->P.c.in_features_graph)
        return set_error(RAMP_ERR_BAD_ARG, "policy: graph_features row stride %lld is below in_features_graph (%d)", (long long)gf_stride,
                         p->P.c.in_features_graph);
    if (n < 0) return set_error(RAMP_ERR_BAD_ARG, "policy: %d rows", n);
    CUDA_TRY(cudaSetDevice(p->device));
    if (!p->ev_done) CUDA_TRY(create(p->ev_done, cudaEventDisableTiming));
    return RAMP_OK;
}

int check_learner_config(const ramp_impala_config_t* cfg) {
    if (!cfg) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (!(cfg->vtrace_clip_rho_threshold > 0) || !(cfg->vtrace_clip_pg_rho_threshold > 0) || !(cfg->lr >= 0) || !(cfg->adam_eps > 0))
        return set_error(RAMP_ERR_BAD_ARG, "impala: the clip thresholds and adam_eps must be > 0, lr >= 0");
    if (cfg->rollout_fragment_length < 0 || cfg->train_batch_size < 1)
        return set_error(RAMP_ERR_BAD_ARG, "impala: rollout_fragment_length must be >= 0, train_batch_size >= 1");
    return RAMP_OK;
}

int check_learner_config(const ramp_pg_config_t* cfg) {
    if (!cfg) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (!(cfg->gamma >= 0) || !(cfg->lr >= 0) || !(cfg->adam_eps > 0)) return set_error(RAMP_ERR_BAD_ARG, "pg: gamma and lr must be >= 0, adam_eps > 0");
    return RAMP_OK;
}

// the opening of every learn call: the algorithm's own configuration check, then a trajectory of at least n_steps recorded from
// eng's environment; the messages start with `tag`.  Leaves the policy's device current and the engine stream in *st.
template <class Cfg>
int learn_begin(ramp_policy* p, ramp_engine_t* eng, const Cfg* cfg, int32_t n_steps, const char* tag, ramp_env_buffers_t* eb,
                cudaStream_t* st) {
    if (!p || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_learner_config(cfg);
    if (rc != RAMP_OK || (rc = ramp_env_buffers(eng, eb)) != RAMP_OK) return rc;
    if (n_steps < 1 || n_steps > p->traj_n)
        return set_error(RAMP_ERR_BAD_ARG, "%s: %d steps asked of a trajectory with %d recorded", tag, n_steps, p->traj_n);
    if (eb->n_episodes != p->traj_b || eb->n_actions != p->traj_a)
        return set_error(RAMP_ERR_BAD_ARG, "%s: the trajectory was recorded from another environment", tag);
    CUDA_TRY(cudaSetDevice(p->device));
    *st = ramp_internal_stream(eng);
    return RAMP_OK;
}

// GAE (ramp_ppo_gae_kernel) over the trajectory's first T steps into the train batch b_*, on `st`.  boot: the value of the state
// after the last step; nullptr: no critic (PG's discounted returns: V = 0, a 0 bootstrap)
int launch_gae(ramp_policy* p, cudaStream_t st, int32_t T, int32_t B, double gamma, double lambda, int32_t standardize, const float* boot) {
    GaeArgs ge{};
    ge.T = T; ge.B = B; ge.A = p->P.c.n_actions; ge.n_models = p->P.c.n_models; ge.standardize = standardize;
    ge.gamma = gamma; ge.lambda = lambda;
    ge.t_obs = p->t_obs.get(); ge.t_model = p->t_model.get(); ge.t_mask = p->t_mask.get(); ge.t_action = p->t_action.get();
    ge.t_logp = p->t_logp.get(); ge.t_value = boot ? p->t_value.get() : nullptr; ge.t_reward = p->t_reward.get(); ge.t_done = p->t_done.get();
    ge.boot = boot; ge.adv64 = p->L.b_adv64.get();
    ge.obs = p->L.b_obs.get(); ge.model = p->L.b_model.get(); ge.mask = p->L.b_mask.get(); ge.action = p->L.b_action.get(); ge.logp = p->L.b_logp.get();
    ge.adv = p->L.b_adv.get(); ge.vt = p->L.b_vt.get(); ge.n_rows = p->L.n_rows.get();
    ramp_ppo_gae_kernel<<<1, 1024, 0, st>>>(ge);
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

// clip_grad_norm_ and torch.optim.Adam at cfg's settings on the policy's gradient, moments and step count, for minibatches of mb
// rows of a batch of *n_rows rows; the caller sets the minibatch's start and where its statistics go
template <class Cfg>
AdamArgs adam_args(ramp_policy* p, const Cfg& cfg, const int32_t* n_rows, int32_t mb) {
    AdamArgs aa{};
    aa.lr = cfg.lr; aa.beta1 = cfg.adam_beta1; aa.beta2 = cfg.adam_beta2;
    aa.beta2_f = (float)cfg.adam_beta2; aa.one_m_beta1 = (float)(1.0 - cfg.adam_beta1); aa.one_m_beta2 = (float)(1.0 - cfg.adam_beta2);
    aa.eps = (float)cfg.adam_eps;
    aa.max_norm = (float)cfg.grad_clip; aa.n_rows = n_rows; aa.mb = mb; aa.step = p->L.step.get();
    aa.m = p->L.adam_m.get(); aa.v = p->L.adam_v.get(); aa.grad = p->L.grad.get(); aa.norm_part = p->L.norm_part.get(); aa.w = p->d_w.get();
    return aa;
}

// one Adam step on `st`: it reads the step count the previous step wrote
int launch_adam(ramp_policy* p, AdamArgs aa, cudaStream_t st) {
    aa.parity = p->L.parity; p->L.parity ^= 1;
    ramp_adam_kernel<<<LRN_GRID, 256, 0, st>>>(aa, p->n_weights);
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

// the end of the gradient calls on host rows (stream 0): the gradient and n_stats statistics from `stats` (either out may be nullptr)
int host_batch_end(ramp_policy* p, float* grad_out, double* stats_out, const double* stats, int n_stats) {
    CUDA_TRY(cudaStreamSynchronize(0));
    if (grad_out) CUDA_TRY(cudaMemcpy(grad_out, p->L.grad.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToHost));
    if (stats_out) CUDA_TRY(cudaMemcpy(stats_out, stats, sizeof(double) * n_stats, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

// IMPALA's per-row arrays for K groups of n fragment rows, and statistics for `steps` SGD steps of K sets
int ensure_impala(LearnerBuffers& L, const ramp_policy_config_t& c, int32_t n, int32_t steps) {
    const size_t K = L.K, A = c.n_actions;
    if (n > L.icap) {
        L.icap = 0;
        CUDA_TRY(alloc_each(K * n, L.i_blogp, L.i_tvalue, L.i_tlogp, L.i_log_rho, L.i_vs, L.i_pg, L.i_model, L.i_action,
                            L.i_actx, L.i_lmodel, L.i_done, L.i_reward));
        CUDA_TRY(L.i_obs.alloc(K * n * 11));
        CUDA_TRY(alloc_each(K * n * A, L.i_tlogits, L.i_mask));
        L.icap = n;
    }
    if (!L.i_n_rows.get()) {
        CUDA_TRY(L.i_n_rows.alloc(K));
        CUDA_TRY(L.i_stats.alloc(K * RAMP_IMPALA_STATS_LEN));
    }
    if (steps > L.i_step_cap) {
        L.i_step_cap = 0;
        CUDA_TRY(L.i_step_stats.alloc(K * steps * RAMP_IMPALA_STATS_LEN));
        L.i_step_cap = steps;
    }
    return RAMP_OK;
}

// one IMPALA batch: the fragment rows [row0, row0 + n_frag L) of the i_* arrays, whose model / action / behaviour log p / reward /
// done are set, read either from the environment-style rows (obs_dyn, i_obs) or host graph features.  The embeddings of
// launch_states are current.  Read-out at the current weights -> V-trace -> loss gradient (l_grad, the norm partials) -> the
// step's statistics into `stats`.  ga: the head-gradient launch (its rows, start, row count and inputs), completed here.
int impala_batch(ramp_policy* p, cudaStream_t st, const ramp_impala_config_t& cfg, int32_t L, int32_t row0, int32_t n_frag,
                 const float* obs_dyn, const float* graph_features, const int32_t* model, const uint8_t* mask, const int32_t* action,
                 const float* blogp, const double* reward, const uint8_t* done, GradArgs ga, double* stats) {
    const ramp_policy_config_t& c = p->P.c;
    const size_t A = c.n_actions, r0 = (size_t)row0;
    int rc;
    HeadArgs h{};
    h.n = n_frag * L; h.graph_features = graph_features ? graph_features + r0 * c.in_features_graph : nullptr;
    h.obs_dyn = obs_dyn ? obs_dyn + r0 * 11 : nullptr; h.graph_static = p->d_gstatic.get();
    h.model = model + r0; h.mask = mask + r0 * A; h.emb = p->d_emb.get();
    h.logits = p->L.i_tlogits.get() + r0 * A; h.value = p->L.i_tvalue.get() + r0; h.actions = p->L.i_actx.get() + r0;
    if ((rc = launch_head(p, h, st)) != RAMP_OK) return rc;
    VtraceArgs v{};
    v.L = L; v.n_frag = n_frag; v.row0 = row0; v.A = c.n_actions; v.n_models = c.n_models;
    v.gamma = cfg.gamma; v.clip_rho = cfg.vtrace_clip_rho_threshold; v.clip_pg_rho = cfg.vtrace_clip_pg_rho_threshold;
    v.logits = p->L.i_tlogits.get(); v.value = p->L.i_tvalue.get();
    v.model = model; v.action = action; v.blogp = blogp; v.reward = reward; v.done = done;
    v.tlogp = p->L.i_tlogp.get(); v.log_rho = p->L.i_log_rho.get(); v.vs = p->L.i_vs.get(); v.pg_adv = p->L.i_pg.get(); v.lmodel = p->L.i_lmodel.get();
    ramp_vtrace_kernel<<<(unsigned)((n_frag + 7) / 8), 256, 0, st>>>(v);
    CUDA_TRY(cudaGetLastError());
    ga.impala = 1; ga.shuffle = 0; ga.graph_features = graph_features; ga.obs_dyn = obs_dyn; ga.model = p->L.i_lmodel.get(); ga.mask = mask;
    ga.action = action; ga.adv = p->L.i_pg.get(); ga.vt = p->L.i_vs.get();
    ga.vf_coeff = (float)cfg.vf_loss_coeff; ga.ent_coeff = (float)cfg.entropy_coeff;
    if ((rc = launch_grad(p, ga, st)) != RAMP_OK) return rc;
    ramp_impala_step_stats_kernel<<<1, 1, 0, st>>>(p->L.row_stats.get(), p->L.row_model.get(), ga.mb, row0, p->L.i_log_rho.get(),
                                                   cfg.vf_loss_coeff, cfg.entropy_coeff, p->L.norm_part.get(), stats);
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

}  // namespace

extern "C" {

int64_t ramp_policy_weight_count(const ramp_policy_config_t* cfg) {
    if (!cfg || check_config(*cfg) != RAMP_OK) return -1;
    return layout(*cfg, nullptr);
}

int ramp_policy_create(int device, const ramp_policy_config_t* cfg, ramp_policy_t** out) {
    if (!cfg || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_config(*cfg);
    if (rc != RAMP_OK) return rc;
    CUDA_TRY(cudaSetDevice(device));
    std::unique_ptr<ramp_policy> p(new ramp_policy());
    p->device = device;
    p->P.c = *cfg;
    p->n_weights = layout(*cfg, &p->P);
    p->models.resize(cfg->n_models);
    cudaDeviceProp prop{};
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) p->sm_count = prop.multiProcessorCount;
    p->head_smem = head_smem_floats(*cfg, 8) * sizeof(float);
    if (p->head_smem > 200 * 1024) return set_error(RAMP_ERR_CAPACITY, "policy: the read-out needs %zu B of shared memory (max 200 KiB)", p->head_smem);
    CUDA_TRY(reserve_dynamic_smem((const void*)ramp_policy_head_kernel, p->head_smem));
    CUDA_TRY(p->d_w.alloc(p->n_weights));
    CUDA_TRY(p->d_models.alloc(cfg->n_models));
    CUDA_TRY(p->d_emb.alloc((size_t)cfg->n_models * cfg->out_features_node));
    CUDA_TRY(p->d_gstatic.alloc((size_t)cfg->n_models * 6));
    cudaMemset(p->d_emb.get(), 0, sizeof(float) * (size_t)cfg->n_models * cfg->out_features_node);
    cudaMemset(p->d_gstatic.get(), 0, sizeof(float) * (size_t)cfg->n_models * 6);
    p->P.w = p->d_w.get();
    *out = p.release();
    return RAMP_OK;
}

void ramp_policy_destroy(ramp_policy_t* p) {
    if (!p) return;
    cudaSetDevice(p->device);
    delete p;
}

int ramp_policy_set_weights(ramp_policy_t* p, const float* weights, int64_t n) {
    if (!p || !weights) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n != p->n_weights) return set_error(RAMP_ERR_BAD_ARG, "policy: %lld weights given, the configuration has %lld", (long long)n, (long long)p->n_weights);
    CUDA_TRY(cudaSetDevice(p->device));
    CUDA_TRY(cudaDeviceSynchronize());                                    // a running rollout may still read the old set
    CUDA_TRY(cudaMemcpy(p->d_w.get(), weights, sizeof(float) * n, cudaMemcpyHostToDevice));
    p->weights_set = true;
    p->emb_valid = false;
    return RAMP_OK;
}

int ramp_policy_set_model(ramp_policy_t* p, int32_t model, int32_t n_nodes, int32_t n_edges, const float* node_features,
                          const float* edge_features, const int32_t* edges_src, const int32_t* edges_dst, const float* graph_static) {
    if (!p || !node_features || !graph_static || (n_edges > 0 && (!edge_features || !edges_src || !edges_dst)))
        return set_error(RAMP_ERR_BAD_ARG, "null argument");
    const ramp_policy_config_t& c = p->P.c;
    if (model < 0 || model >= c.n_models || n_nodes < 1 || n_edges < 0) return set_error(RAMP_ERR_BAD_ARG, "policy: bad model %d (%d nodes, %d edges)", model, n_nodes, n_edges);
    for (int e = 0; e < n_edges; ++e)
        if (edges_src[e] < 0 || edges_src[e] >= n_nodes || edges_dst[e] < 0 || edges_dst[e] >= n_nodes)
            return set_error(RAMP_ERR_BAD_ARG, "policy: edge %d of model %d names node %d -> %d of %d", e, model, edges_src[e], edges_dst[e], n_nodes);
    CUDA_TRY(cudaSetDevice(p->device));
    HostModel& hm = p->models[model];
    hm.allocs.clear();
    hm.lallocs.clear();
    hm.set = hm.grad_ready = p->L.gmodels_ready = false;
    // incoming-edge lists by destination, in edge order (the order DGL delivers a node's mailbox is not observable through a mean)
    std::vector<int32_t> ptr(n_nodes + 1, 0), ine(n_edges), ins(n_edges);
    for (int e = 0; e < n_edges; ++e) ptr[edges_dst[e] + 1]++;
    for (int v = 0; v < n_nodes; ++v) ptr[v + 1] += ptr[v];
    std::vector<int32_t> cur(ptr.begin(), ptr.end() - 1);
    for (int e = 0; e < n_edges; ++e) { const int at = cur[edges_dst[e]]++; ine[at] = e; ins[at] = edges_src[e]; }
    const int half = c.out_features_msg / 2;
    auto up = [&](const void* src, size_t bytes, const void** dst) -> int {
        hm.allocs.emplace_back();
        CUDA_TRY(hm.allocs.back().alloc(bytes ? bytes : 4));
        void* d = hm.allocs.back().get();
        if (src && bytes) CUDA_TRY(cudaMemcpy(d, src, bytes, cudaMemcpyHostToDevice));
        *dst = d;
        return RAMP_OK;
    };
    int rc;
    ModelDev d{};
    d.n_nodes = n_nodes; d.n_edges = n_edges;
    if ((rc = up(node_features, sizeof(float) * (size_t)n_nodes * c.in_features_node, (const void**)&d.nf))) return rc;
    if ((rc = up(edge_features, sizeof(float) * (size_t)n_edges * c.in_features_edge, (const void**)&d.ef))) return rc;
    if ((rc = up(ptr.data(), sizeof(int32_t) * ptr.size(), (const void**)&d.in_ptr))) return rc;
    if ((rc = up(ine.data(), sizeof(int32_t) * ine.size(), (const void**)&d.in_edge))) return rc;
    if ((rc = up(ins.data(), sizeof(int32_t) * ins.size(), (const void**)&d.in_src))) return rc;
    if ((rc = up(nullptr, sizeof(float) * (size_t)n_nodes * POL_MAX_DIM, (const void**)&d.z0))) return rc;
    if ((rc = up(nullptr, sizeof(float) * (size_t)n_nodes * POL_MAX_DIM, (const void**)&d.z1))) return rc;
    if ((rc = up(nullptr, sizeof(float) * (size_t)n_nodes * half, (const void**)&d.hn))) return rc;
    if ((rc = up(nullptr, sizeof(float) * (size_t)n_edges * half, (const void**)&d.he))) return rc;
    // outgoing-edge lists by source, in edge order: the backward gathers a node's message gradients through them
    std::vector<int32_t> optr(n_nodes + 1, 0), oute(n_edges);
    for (int e = 0; e < n_edges; ++e) optr[edges_src[e] + 1]++;
    for (int v = 0; v < n_nodes; ++v) optr[v + 1] += optr[v];
    std::vector<int32_t> ocur(optr.begin(), optr.end() - 1);
    for (int e = 0; e < n_edges; ++e) oute[ocur[edges_src[e]]++] = e;
    GradModelDev g{};
    if ((rc = up(optr.data(), sizeof(int32_t) * optr.size(), (const void**)&g.out_ptr))) return rc;
    if ((rc = up(oute.data(), sizeof(int32_t) * oute.size(), (const void**)&g.out_edge))) return rc;
    CUDA_TRY(cudaMemcpy(p->d_gstatic.get() + (size_t)model * 6, graph_static, sizeof(float) * 6, cudaMemcpyHostToDevice));
    hm.g = g;
    hm.d = d;
    CUDA_TRY(cudaMemcpy(p->d_models.get() + model, &d, sizeof(ModelDev), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaDeviceSynchronize());                                    // a kernel on any stream may read the table next
    hm.set = true;
    p->emb_valid = false;
    return RAMP_OK;
}

int ramp_policy_embed(ramp_policy_t* p, float* embeddings_out) {
    if (!p) return set_error(RAMP_ERR_BAD_ARG, "null policy");
    CUDA_TRY(cudaSetDevice(p->device));
    int rc;
    if ((rc = fence_in(p, 0)) != RAMP_OK || (rc = launch_embed(p, 0)) != RAMP_OK) return rc;
    CUDA_TRY(cudaStreamSynchronize(0));
    if (embeddings_out)
        CUDA_TRY(cudaMemcpy(embeddings_out, p->d_emb.get(), sizeof(float) * (size_t)p->P.c.n_models * p->P.c.out_features_node, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_policy_forward(ramp_policy_t* p, int32_t n, const int32_t* model, const float* graph_features, const uint8_t* action_mask,
                        float* logits_out, float* value_out) {
    return head_on_host(p, n, model, graph_features, action_mask, 0, 0, logits_out, value_out, nullptr, nullptr);
}

int ramp_policy_decide(ramp_policy_t* p, int32_t n, const int32_t* model, const float* graph_features, const uint8_t* action_mask,
                       int32_t sample, uint64_t seed, float* logits_out, float* value_out, float* logp_out, int32_t* actions_out) {
    return head_on_host(p, n, model, graph_features, action_mask, sample, seed, logits_out, value_out, logp_out, actions_out);
}

int ramp_policy_act(ramp_policy_t* p, ramp_engine_t* eng, int32_t sample, uint64_t seed) {
    if (!p || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    ramp_env_buffers_t eb{};
    int rc = ramp_env_buffers(eng, &eb);
    if (rc != RAMP_OK) return rc;
    const ramp_policy_config_t& c = p->P.c;
    if (ramp_internal_device(eng) != p->device) return set_error(RAMP_ERR_BAD_ARG, "policy and engine live on different devices");
    if (eb.n_actions != c.n_actions) return set_error(RAMP_ERR_BAD_ARG, "policy has %d actions, the environment %d", c.n_actions, eb.n_actions);
    if (c.in_features_graph != 17) return set_error(RAMP_ERR_BAD_ARG, "the environment emits 17 graph features, the policy expects %d", c.in_features_graph);
    if (eb.n_models > c.n_models) return set_error(RAMP_ERR_BAD_ARG, "the environment has %d job types, the policy %d", eb.n_models, c.n_models);
    CUDA_TRY(cudaSetDevice(p->device));
    cudaStream_t st = ramp_internal_stream(eng);
    int launches = 1;
    if ((rc = fence_in(p, st)) != RAMP_OK) return rc;
    if (!p->emb_valid) { if ((rc = launch_embed(p, st)) != RAMP_OK) return rc; ++launches; }
    if ((rc = ensure_outputs(p, eb.n_episodes)) != RAMP_OK) return rc;
    HeadArgs a{};
    a.n = eb.n_episodes; a.obs_dyn = eb.obs_dynamic; a.graph_static = p->d_gstatic.get(); a.model = eb.queued_model; a.done = eb.done;
    a.mask = eb.action_mask; a.emb = p->d_emb.get(); a.logits = p->d_logits.get(); a.value = p->d_value.get(); a.logp = p->d_logp.get(); a.actions = eb.actions;
    a.sample = sample; a.seed = seed ^ (0x9E3779B97F4A7C15ull * (++p->act_calls));
    if ((rc = launch_head(p, a, st)) != RAMP_OK || (rc = fence_out(p, st)) != RAMP_OK) return rc;
    p->act_n = eb.n_episodes;
    ramp_internal_count_launches(eng, launches);
    return RAMP_OK;
}

int ramp_policy_read(ramp_policy_t* p, ramp_engine_t* eng, float* logits_out, float* value_out, float* logp_out, int32_t* actions_out) {
    if (!p || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    ramp_env_buffers_t eb{};
    int rc = ramp_env_buffers(eng, &eb);
    if (rc != RAMP_OK) return rc;
    if (eb.n_episodes != p->act_n) return set_error(RAMP_ERR_BAD_ARG, "policy: nothing to read (ramp_policy_act was not called for this environment)");
    cudaStream_t st = ramp_internal_stream(eng);
    const size_t B = (size_t)eb.n_episodes;
    if (logits_out) CUDA_TRY(cudaMemcpyAsync(logits_out, p->d_logits.get(), sizeof(float) * B * p->P.c.n_actions, cudaMemcpyDeviceToHost, st));
    if (value_out) CUDA_TRY(cudaMemcpyAsync(value_out, p->d_value.get(), sizeof(float) * B, cudaMemcpyDeviceToHost, st));
    if (logp_out) CUDA_TRY(cudaMemcpyAsync(logp_out, p->d_logp.get(), sizeof(float) * B, cudaMemcpyDeviceToHost, st));
    if (actions_out) CUDA_TRY(cudaMemcpyAsync(actions_out, eb.actions, sizeof(int32_t) * B, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

void* ramp_pinned_alloc(size_t bytes) {
    void* ptr = nullptr;
    if (cudaMallocHost(&ptr, bytes ? bytes : 1) != cudaSuccess) { set_error(RAMP_ERR_CUDA, "cudaMallocHost(%zu) failed", bytes); return nullptr; }
    return ptr;
}

void ramp_pinned_free(void* ptr) { if (ptr) cudaFreeHost(ptr); }

int ramp_policy_trajectory_begin(ramp_policy_t* p, ramp_engine_t* eng, int32_t horizon) {
    if (!p || !eng || horizon < 1) return set_error(RAMP_ERR_BAD_ARG, "policy: bad trajectory horizon");
    ramp_env_buffers_t eb{};
    int rc = ramp_env_buffers(eng, &eb);
    if (rc != RAMP_OK) return rc;
    CUDA_TRY(cudaSetDevice(p->device));
    p->traj_n = 0;
    if (horizon == p->traj_h && eb.n_episodes == p->traj_b && eb.n_actions == p->traj_a) return RAMP_OK;
    CUDA_TRY(cudaStreamSynchronize(ramp_internal_stream(eng)));
    p->traj_h = 0;                        // until every buffer has the new size
    const size_t n = (size_t)horizon * (size_t)eb.n_episodes;
    CUDA_TRY(alloc_each(n, p->t_model, p->t_action, p->t_logp, p->t_value, p->t_reward, p->t_done));
    CUDA_TRY(p->t_obs.alloc(11 * n));
    CUDA_TRY(p->t_mask.alloc((size_t)eb.n_actions * n));
    p->traj_h = horizon; p->traj_b = eb.n_episodes; p->traj_a = eb.n_actions;
    return RAMP_OK;
}

int ramp_policy_trajectory_record(ramp_policy_t* p, ramp_engine_t* eng, int32_t t, int32_t phase) {
    if (!p || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (p->traj_h < 1 || t < 0 || t >= p->traj_h) return set_error(RAMP_ERR_BAD_ARG, "policy: trajectory slot %d outside [0, %d)", t, p->traj_h);
    ramp_env_buffers_t eb{};
    int rc = ramp_env_buffers(eng, &eb);
    if (rc != RAMP_OK) return rc;
    if (eb.n_episodes != p->traj_b || eb.n_actions != p->traj_a || eb.n_episodes != p->act_n)
        return set_error(RAMP_ERR_BAD_ARG, "policy: the trajectory was set up for another environment, or ramp_policy_act was not called");
    cudaStream_t st = ramp_internal_stream(eng);
    const size_t B = (size_t)eb.n_episodes, o = (size_t)t * B;
    // phase 0: after ramp_policy_act, before the environment steps -- what the policy saw and decided;
    // phase 1: after the environment stepped -- what came back
    TrajArgs a{};
    a.B = eb.n_episodes; a.A = p->traj_a; a.phase = phase;
    a.obs = eb.obs_dynamic; a.model = eb.queued_model; a.mask = eb.action_mask; a.action = eb.actions; a.logp = p->d_logp.get(); a.value = p->d_value.get();
    a.reward = eb.reward; a.done = eb.done;
    a.t_obs = p->t_obs.get() + o * 11; a.t_model = p->t_model.get() + o; a.t_mask = p->t_mask.get() + o * p->traj_a; a.t_action = p->t_action.get() + o;
    a.t_logp = p->t_logp.get() + o; a.t_value = p->t_value.get() + o; a.t_reward = p->t_reward.get() + o; a.t_done = p->t_done.get() + o;
    ramp_trajectory_record_kernel<<<(unsigned)((B + 127) / 128), 128, 0, st>>>(a);
    CUDA_TRY(cudaGetLastError());
    if (phase == 1 && t == p->traj_n) p->traj_n = t + 1;
    ramp_internal_count_launches(eng, 1);
    return RAMP_OK;
}

int ramp_policy_trajectory_read(ramp_policy_t* p, ramp_engine_t* eng, int32_t n_steps, float* obs_dynamic_out, int32_t* model_out,
                                uint8_t* action_mask_out, int32_t* action_out, float* logp_out, float* value_out, double* reward_out,
                                uint8_t* done_out) {
    if (!p || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n_steps < 1 || n_steps > p->traj_h) return set_error(RAMP_ERR_BAD_ARG, "policy: %d steps asked of a trajectory of %d", n_steps, p->traj_h);
    cudaStream_t st = ramp_internal_stream(eng);
    const size_t n = (size_t)n_steps * (size_t)p->traj_b;
    if (obs_dynamic_out) CUDA_TRY(cudaMemcpyAsync(obs_dynamic_out, p->t_obs.get(), sizeof(float) * 11 * n, cudaMemcpyDeviceToHost, st));
    if (model_out) CUDA_TRY(cudaMemcpyAsync(model_out, p->t_model.get(), sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    if (action_mask_out) CUDA_TRY(cudaMemcpyAsync(action_mask_out, p->t_mask.get(), (size_t)p->traj_a * n, cudaMemcpyDeviceToHost, st));
    if (action_out) CUDA_TRY(cudaMemcpyAsync(action_out, p->t_action.get(), sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    if (logp_out) CUDA_TRY(cudaMemcpyAsync(logp_out, p->t_logp.get(), sizeof(float) * n, cudaMemcpyDeviceToHost, st));
    if (value_out) CUDA_TRY(cudaMemcpyAsync(value_out, p->t_value.get(), sizeof(float) * n, cudaMemcpyDeviceToHost, st));
    if (reward_out) CUDA_TRY(cudaMemcpyAsync(reward_out, p->t_reward.get(), sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    if (done_out) CUDA_TRY(cudaMemcpyAsync(done_out, p->t_done.get(), n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

int ramp_policy_get_weights(ramp_policy_t* p, float* out) {
    if (!p || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (!p->weights_set) return set_error(RAMP_ERR_BAD_ARG, "policy: no weights (ramp_policy_set_weights)");
    CUDA_TRY(cudaSetDevice(p->device));
    CUDA_TRY(cudaDeviceSynchronize());                                    // a learn call may still be updating them
    CUDA_TRY(cudaMemcpy(out, p->d_w.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_policy_backward(ramp_policy_t* p, int32_t n, const int32_t* model, const float* graph_features, const uint8_t* action_mask,
                         const float* grad_logits, const float* grad_value, float* grad_weights_out) {
    if (!p || !model || !graph_features || !action_mask || !grad_logits || !grad_value || !grad_weights_out)
        return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n < 1) return set_error(RAMP_ERR_BAD_ARG, "policy: backward of %d rows", n);
    CUDA_TRY(cudaSetDevice(p->device));
    int rc;
    if ((rc = prepare_learner(p, 0, n)) ||
        (rc = upload_host_batch(p, n, model, graph_features, action_mask, grad_logits, grad_value, nullptr, nullptr, nullptr, nullptr)) ||
        (rc = launch_backward(p, 0, n, false)))
        return rc;
    return host_batch_end(p, grad_weights_out, nullptr, nullptr, 0);
}

int ramp_policy_set_weights_device(ramp_policy_t* p, const float* weights, int64_t n, void* stream) {
    if (!p || !weights) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n != p->n_weights) return set_error(RAMP_ERR_BAD_ARG, "policy: %lld weights given, the configuration has %lld", (long long)n, (long long)p->n_weights);
    CUDA_TRY(cudaSetDevice(p->device));
    if (!p->ev_done) CUDA_TRY(create(p->ev_done, cudaEventDisableTiming));
    cudaStream_t st = (cudaStream_t)stream;
    int rc;
    if ((rc = fence_in(p, st)) != RAMP_OK) return rc;                    // a queued call may still read the old set
    CUDA_TRY(cudaMemcpyAsync(p->d_w.get(), weights, sizeof(float) * n, cudaMemcpyDeviceToDevice, st));
    p->weights_set = true;
    p->emb_valid = false;
    return fence_out(p, st);
}

// the embeddings remade into d_emb on `st` when stale.  Once a backward has set up the learner, they are remade by the gradient
// kernel's forward instance: the same bits, and its kept states spare the next backward a second pass over the MeanPool rounds
// (the fused learners do the same)
int refresh_embeddings(ramp_policy* p, cudaStream_t st) {
    if (p->emb_valid) return RAMP_OK;
    if (p->L.ready && p->L.gmodels_ready) {
        int rc = launch_states(p, st, nullptr, 0, p->d_emb.get());
        if (rc != RAMP_OK) return rc;
        p->emb_valid = true;
        return RAMP_OK;
    }
    return launch_embed(p, st);
}

int ramp_policy_forward_device(ramp_policy_t* p, void* stream, int32_t n, const void* model, int32_t model_dtype,
                               const float* graph_features, int64_t graph_features_stride, const uint8_t* action_mask,
                               float* logits_out, float* value_out) {
    if (!p || !logits_out || !value_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    bool capturing = false;
    int rc = capture_status(st, &capturing);
    if (rc != RAMP_OK) return rc;
    if (capturing) {
        // a replay runs no host code: the weights, embeddings and staging are what eager calls left, and the graph reads them
        // at their addresses.  The fencing event is not used: the graph's replays are ordered on the capturing stream's successor
        if (!p->emb_valid || !p->ev_done)
            return set_error(RAMP_ERR_BAD_ARG, "CUDA-graph capture refused: the policy's embeddings are stale and would be remade "
                             "inside the graph; call refresh() (ramp_policy_refresh_device) or an eager forward first");
        if (n > p->fcap)
            return set_error(RAMP_ERR_BAD_ARG, "CUDA-graph capture refused: %d rows are more than any eager forward staged (%d); the "
                             "staging would have to grow", n, p->fcap);
    }
    rc = device_call_ready(p, n, model, model_dtype, graph_features, graph_features_stride, action_mask);
    if (rc != RAMP_OK || n == 0) return rc;
    if ((rc = stage_forward(p, n)) != RAMP_OK || (!capturing && (rc = fence_in(p, st)) != RAMP_OK) ||
        (rc = launch_ingest(p, st, n, model, model_dtype, graph_features, graph_features_stride, action_mask, nullptr, nullptr)) != RAMP_OK ||
        (rc = refresh_embeddings(p, st)) != RAMP_OK)
        return rc;
    if ((rc = launch_forward(p, st, n, 0, 0, logits_out, value_out, nullptr)) != RAMP_OK) return rc;
    if (capturing) p->fwd_captured = true;
    return capturing ? RAMP_OK : fence_out(p, st);
}

int ramp_policy_refresh_device(ramp_policy_t* p, void* stream) {
    if (!p) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    bool capturing = false;
    int rc = capture_status(st, &capturing);
    if (rc != RAMP_OK) return rc;
    if (capturing) return set_error(RAMP_ERR_BAD_ARG, "ramp_policy_refresh_device cannot be captured: it runs before a replay, eagerly");
    CUDA_TRY(cudaSetDevice(p->device));
    if (p->emb_valid) return RAMP_OK;
    if (!p->ev_done) CUDA_TRY(create(p->ev_done, cudaEventDisableTiming));
    if ((rc = fence_in(p, st)) != RAMP_OK || (rc = refresh_embeddings(p, st)) != RAMP_OK) return rc;
    return fence_out(p, st);
}

int ramp_policy_backward_device(ramp_policy_t* p, void* stream, int32_t n, const void* model, int32_t model_dtype,
                                const float* graph_features, int64_t graph_features_stride, const uint8_t* action_mask,
                                const float* grad_logits, const float* grad_value, float* grad_weights_out) {
    if (!p || !grad_logits || !grad_value || !grad_weights_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    bool capturing = false;
    int rc = capture_status(st, &capturing);
    if (rc != RAMP_OK) return rc;
    if (capturing) return set_error(RAMP_ERR_BAD_ARG, "CUDA-graph capture refused: the policy's backward is not capturable");
    rc = device_call_ready(p, n, model, model_dtype, graph_features, graph_features_stride, action_mask);
    if (rc != RAMP_OK) return rc;
    if (n < 1) return set_error(RAMP_ERR_BAD_ARG, "policy: backward of %d rows", n);
    if ((rc = prepare_learner(p, st, n)) != RAMP_OK || (rc = stage_host_batch(p, n)) != RAMP_OK ||
        (rc = launch_ingest(p, st, n, model, model_dtype, graph_features, graph_features_stride, action_mask, grad_logits, grad_value)) != RAMP_OK ||
        (rc = launch_backward(p, st, n, true)) != RAMP_OK)
        return rc;
    CUDA_TRY(cudaMemcpyAsync(grad_weights_out, p->L.grad.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToDevice, st));
    return fence_out(p, st);
}

int ramp_ppo_loss_grad(ramp_policy_t* p, const ramp_ppo_config_t* cfg, int32_t n, const int32_t* model, const float* graph_features,
                       const uint8_t* action_mask, const int32_t* action, const float* old_logits, const float* advantage,
                       const float* value_target, float* grad_out, double* stats_out) {
    if (!p || !model || !graph_features || !action_mask || !action || !old_logits || !advantage || !value_target)
        return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_learner_config(cfg);
    if (rc != RAMP_OK) return rc;
    if (n < 1) return set_error(RAMP_ERR_BAD_ARG, "ppo: loss of %d rows", n);
    CUDA_TRY(cudaSetDevice(p->device));
    if ((rc = prepare_learner(p, 0, n)) ||
        (rc = upload_host_batch(p, n, model, graph_features, action_mask, nullptr, nullptr, action, old_logits, advantage, value_target)))
        return rc;
    GradArgs ga = host_batch_args(p, n);
    ga.action = p->h_action.get(); ga.old_logits = p->h_old.get(); ga.adv = p->h_adv.get(); ga.vt = p->h_vt.get();
    ppo_terms(ga, *cfg);
    if ((rc = launch_states(p, 0, nullptr, 0, nullptr)) != RAMP_OK || (rc = launch_grad(p, ga, 0)) != RAMP_OK) return rc;
    ramp_ppo_minibatch_stats_kernel<<<1, 1>>>(p->L.row_stats.get(), n, ga.vf_coeff, ga.ent_coeff, ga.kl_coeff, p->L.norm_part.get(), p->L.stats.get());
    CUDA_TRY(cudaGetLastError());
    return host_batch_end(p, grad_out, stats_out, p->L.stats.get(), RAMP_PPO_STATS_LEN);
}

int ramp_policy_learn(ramp_policy_t* p, ramp_engine_t* eng, int32_t n_steps, const ramp_ppo_config_t* cfg, double* stats_out) {
    ramp_env_buffers_t eb{};
    cudaStream_t st;
    int rc = learn_begin(p, eng, cfg, n_steps, "ppo", &eb, &st);
    if (rc != RAMP_OK) return rc;
    const int32_t B = eb.n_episodes, rows = n_steps * B, mb = cfg->sgd_minibatch_size, n_mb = (rows + mb - 1) / mb;
    if ((rc = prepare_learner(p, st, mb)) || (rc = ensure_batch(p->L, p->P.c, rows)) || (rc = ensure_ppo(p->L, B, n_mb))) return rc;
    int launches = 2;                                                   // GAE, old logits
    // 1. the value of the state after the last step (RLlib's truncate_episodes bootstrap): when the trajectory goes on, the value
    //    act recorded in slot n_steps; after its last recorded slot, the environment's current state, by the head kernel on its
    //    buffers -- not through ramp_policy_act, which mixes its call count into the seed and writes the action buffer
    const float* boot = p->t_value.get() + (size_t)n_steps * B;
    if (n_steps == p->traj_n) {
        HeadArgs hb{};
        hb.n = B; hb.obs_dyn = eb.obs_dynamic; hb.graph_static = p->d_gstatic.get(); hb.model = eb.queued_model; hb.done = eb.done;
        hb.mask = eb.action_mask; hb.emb = p->d_emb.get(); hb.value = p->L.boot.get(); hb.actions = p->L.boot_act.get();
        if ((rc = launch_head(p, hb, st)) != RAMP_OK) return rc;
        boot = p->L.boot.get();
        ++launches;
    }
    // 2. GAE, the live rows t-major, standardised advantages
    if ((rc = launch_gae(p, st, n_steps, B, cfg->gamma, cfg->lambda, cfg->standardize_advantages, boot)) != RAMP_OK) return rc;
    // 3. the collection weights' logits of every row: the head kernel again, so they are act's bits
    HeadArgs ho{};
    ho.n = rows; ho.obs_dyn = p->L.b_obs.get(); ho.graph_static = p->d_gstatic.get(); ho.model = p->L.b_model.get(); ho.mask = p->L.b_mask.get();
    ho.emb = p->d_emb.get(); ho.logits = p->L.b_old.get(); ho.value = p->L.b_value.get(); ho.logp = p->L.b_lpx.get(); ho.actions = p->L.b_actx.get();
    if ((rc = launch_head(p, ho, st)) != RAMP_OK) return rc;
    // 4. num_sgd_iter shuffled passes of minibatch updates; a minibatch past the batch's end (its size is on the device) is a no-op
    GradArgs ga{};
    ga.mb = mb; ga.n_rows = p->L.n_rows.get(); ga.shuffle = 1; ga.obs_dyn = p->L.b_obs.get(); ga.model = p->L.b_model.get();
    ga.mask = p->L.b_mask.get(); ga.action = p->L.b_action.get(); ga.old_logits = p->L.b_old.get(); ga.adv = p->L.b_adv.get(); ga.vt = p->L.b_vt.get();
    ppo_terms(ga, *cfg);
    AdamArgs aa = adam_args(p, *cfg, p->L.n_rows.get(), mb);
    aa.row_stats = p->L.row_stats.get(); aa.vf_coeff = ga.vf_coeff; aa.ent_coeff = ga.ent_coeff; aa.kl_coeff = ga.kl_coeff;
    for (int pass = 0; pass < cfg->num_sgd_iter; ++pass) {
        ga.key = mix64(cfg->seed ^ mix64((uint64_t)pass + 1));
        ga.logp_old = pass == 0 ? p->L.b_logp_old.get() : nullptr;
        for (int k = 0; k < n_mb; ++k) {
            // the rounds at the current weights, kept for the backward; from the second minibatch on also the embeddings, which
            // the previous update made stale (the first uses those the old logits were computed with)
            ga.start = aa.start = k * mb;
            if ((rc = launch_states(p, st, p->L.n_rows.get(), ga.start, pass || k ? p->d_emb.get() : nullptr)) != RAMP_OK ||
                (rc = launch_grad(p, ga, st)) != RAMP_OK)
                return rc;
            aa.stats = p->L.mb_stats.get() + (size_t)k * RAMP_PPO_STATS_LEN;
            if ((rc = launch_adam(p, aa, st)) != RAMP_OK) return rc;
            launches += 6;
        }
    }
    if (cfg->num_sgd_iter > 0) p->emb_valid = false;
    p->b_rows = rows;
    // 5. the last pass's statistics and the adapted KL coefficient: the call's one read-back
    ramp_ppo_learn_stats_kernel<<<1, 1, 0, st>>>(p->L.mb_stats.get(), cfg->num_sgd_iter > 0 ? n_mb : 0, (float)cfg->kl_coeff,
                                                 (float)cfg->kl_target, p->L.n_rows.get(), p->L.stats.get());
    CUDA_TRY(cudaGetLastError());
    ramp_internal_count_launches(eng, launches + 1);
    if (stats_out) CUDA_TRY(cudaMemcpyAsync(stats_out, p->L.stats.get(), sizeof(double) * RAMP_PPO_STATS_LEN, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

int ramp_policy_train_batch_read(ramp_policy_t* p, ramp_engine_t* eng, int32_t* n_out, int32_t* model_out, int32_t* action_out,
                                 float* logp_out, float* logp_old_out, float* advantage_out, float* value_target_out) {
    if (!p || !eng || !n_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (p->b_rows < 1) return set_error(RAMP_ERR_BAD_ARG, "ppo: no train batch (ramp_policy_learn / ramp_policy_learn_pg)");
    cudaStream_t st = ramp_internal_stream(eng);
    CUDA_TRY(cudaMemcpyAsync(n_out, p->L.n_rows.get(), sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    const size_t n = (size_t)*n_out;
    if (model_out) CUDA_TRY(cudaMemcpyAsync(model_out, p->L.b_model.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    if (action_out) CUDA_TRY(cudaMemcpyAsync(action_out, p->L.b_action.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    if (logp_out) CUDA_TRY(cudaMemcpyAsync(logp_out, p->L.b_logp.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    if (logp_old_out) CUDA_TRY(cudaMemcpyAsync(logp_old_out, p->L.b_logp_old.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    if (advantage_out) CUDA_TRY(cudaMemcpyAsync(advantage_out, p->L.b_adv.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    if (value_target_out) CUDA_TRY(cudaMemcpyAsync(value_target_out, p->L.b_vt.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

int ramp_policy_learner_state(ramp_policy_t* p, float* exp_avg_out, float* exp_avg_sq_out, int32_t* step_out) {
    if (!p) return set_error(RAMP_ERR_BAD_ARG, "null policy");
    CUDA_TRY(cudaSetDevice(p->device));
    if (!p->L.ready) {
        if (exp_avg_out) memset(exp_avg_out, 0, sizeof(float) * p->n_weights);
        if (exp_avg_sq_out) memset(exp_avg_sq_out, 0, sizeof(float) * p->n_weights);
        if (step_out) *step_out = 0;
        return RAMP_OK;
    }
    CUDA_TRY(cudaDeviceSynchronize());                                    // a learn call may still be updating them
    if (exp_avg_out) CUDA_TRY(cudaMemcpy(exp_avg_out, p->L.adam_m.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToHost));
    if (exp_avg_sq_out) CUDA_TRY(cudaMemcpy(exp_avg_sq_out, p->L.adam_v.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToHost));
    if (step_out) CUDA_TRY(cudaMemcpy(step_out, p->L.step.get() + p->L.parity, sizeof(int32_t), cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_policy_learner_reset(ramp_policy_t* p) {
    if (!p) return set_error(RAMP_ERR_BAD_ARG, "null policy");
    CUDA_TRY(cudaSetDevice(p->device));
    if (!p->L.ready) return RAMP_OK;
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemset(p->L.adam_m.get(), 0, sizeof(float) * p->n_weights));
    CUDA_TRY(cudaMemset(p->L.adam_v.get(), 0, sizeof(float) * p->n_weights));
    CUDA_TRY(cudaMemset(p->L.step.get(), 0, sizeof(int32_t) * 2));
    return RAMP_OK;
}

int ramp_policy_set_learner_state(ramp_policy_t* p, const float* exp_avg, const float* exp_avg_sq, int64_t n, int32_t step) {
    if (!p || !exp_avg || !exp_avg_sq) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n != p->n_weights)
        return set_error(RAMP_ERR_BAD_ARG, "policy: a learner state of %lld weights given, the configuration has %lld", (long long)n, (long long)p->n_weights);
    if (step < 0) return set_error(RAMP_ERR_BAD_ARG, "policy: Adam step count %d < 0", step);
    CUDA_TRY(cudaSetDevice(p->device));
    int rc = ensure_learner(p->L, p->n_weights, (size_t)p->P.c.n_models * gnn_weight_count(p));
    if (rc != RAMP_OK) return rc;
    CUDA_TRY(cudaDeviceSynchronize());                                    // a learn call may still be updating them
    CUDA_TRY(cudaMemcpy(p->L.adam_m.get(), exp_avg, sizeof(float) * n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(p->L.adam_v.get(), exp_avg_sq, sizeof(float) * n, cudaMemcpyHostToDevice));
    const int32_t steps[2] = {step, step};                              // whichever parity the next step reads
    CUDA_TRY(cudaMemcpy(p->L.step.get(), steps, sizeof(steps), cudaMemcpyHostToDevice));
    return RAMP_OK;
}

int ramp_policy_get_act_count(ramp_policy_t* p, uint64_t* out) {
    if (!p || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    *out = p->act_calls;
    return RAMP_OK;
}

int ramp_policy_set_act_count(ramp_policy_t* p, uint64_t n) {
    if (!p) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    p->act_calls = n;
    return RAMP_OK;
}

int ramp_impala_loss_grad(ramp_policy_t* p, const ramp_impala_config_t* cfg, int32_t n_fragments, int32_t fragment_length,
                          const int32_t* model, const float* graph_features, const uint8_t* action_mask, const int32_t* action,
                          const float* behaviour_logp, const double* reward, const uint8_t* done, float* grad_out,
                          double* stats_out, float* vs_out, float* pg_adv_out, float* log_rho_out) {
    if (!p || !model || !graph_features || !action_mask || !action || !behaviour_logp || !reward || !done)
        return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_learner_config(cfg);
    if (rc != RAMP_OK) return rc;
    if (n_fragments < 1 || fragment_length < 1 || (int64_t)n_fragments * fragment_length > INT32_MAX)
        return set_error(RAMP_ERR_BAD_ARG, "impala: loss of %d fragments of %d rows", n_fragments, fragment_length);
    const int32_t n = n_fragments * fragment_length;
    CUDA_TRY(cudaSetDevice(p->device));
    if ((rc = prepare_learner(p, 0, n)) || (rc = ensure_impala(p->L, p->P.c, n, 1)) ||
        (rc = upload_host_batch(p, n, model, graph_features, action_mask, nullptr, nullptr, action, nullptr, nullptr, nullptr)))
        return rc;
    CUDA_TRY(cudaMemcpy(p->L.i_blogp.get(), behaviour_logp, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(p->L.i_reward.get(), reward, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(p->L.i_done.get(), done, (size_t)n, cudaMemcpyHostToDevice));
    if ((rc = launch_states(p, 0, nullptr, 0, nullptr)) != RAMP_OK) return rc;
    GradArgs ga = host_batch_args(p, n);
    if ((rc = impala_batch(p, 0, *cfg, fragment_length, 0, n_fragments, nullptr, p->h_gf.get(), p->h_model.get(), p->h_mask.get(),
                           p->h_action.get(), p->L.i_blogp.get(), p->L.i_reward.get(), p->L.i_done.get(), ga, p->L.i_stats.get())) != RAMP_OK)
        return rc;
    CUDA_TRY(cudaMemsetAsync(p->L.i_stats.get() + RAMP_IMPALA_SGD_STEPS, 0, sizeof(double), 0));
    if ((rc = host_batch_end(p, grad_out, stats_out, p->L.i_stats.get(), RAMP_IMPALA_STATS_LEN)) != RAMP_OK) return rc;
    p->L.i_rows = n;
    if (vs_out) CUDA_TRY(cudaMemcpy(vs_out, p->L.i_vs.get(), sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
    if (pg_adv_out) CUDA_TRY(cudaMemcpy(pg_adv_out, p->L.i_pg.get(), sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
    if (log_rho_out) CUDA_TRY(cudaMemcpy(log_rho_out, p->L.i_log_rho.get(), sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_policy_learn_impala(ramp_policy_t* p, ramp_engine_t* eng, int32_t n_steps, const ramp_impala_config_t* cfg, double* stats_out) {
    ramp_env_buffers_t eb{};
    cudaStream_t st;
    int rc = learn_begin(p, eng, cfg, n_steps, "impala", &eb, &st);
    if (rc != RAMP_OK) return rc;
    const int32_t L = cfg->rollout_fragment_length ? cfg->rollout_fragment_length : n_steps;
    if (n_steps % L) return set_error(RAMP_ERR_BAD_ARG, "impala: rollout_fragment_length %d does not divide %d steps", L, n_steps);
    if (cfg->train_batch_size < L)
        return set_error(RAMP_ERR_BAD_ARG, "impala: train_batch_size %d is below rollout_fragment_length %d", cfg->train_batch_size, L);
    const ramp_policy_config_t& c = p->P.c;
    const int32_t B = eb.n_episodes, n_frag = (n_steps / L) * B, R = n_steps * B;
    const int32_t F = std::min(cfg->train_batch_size / L, n_frag), mb = F * L, n_sgd = (n_frag + F - 1) / F;
    if ((rc = prepare_learner(p, st, mb)) || (rc = ensure_impala(p->L, p->P.c, R, n_sgd))) return rc;
    // 1. the fragment rows, fragment-major
    ImpalaBatchArgs ba{};
    ba.T = n_steps; ba.B = B; ba.A = c.n_actions; ba.L = L; ba.n_models = c.n_models;
    ba.t_obs = p->t_obs.get(); ba.t_model = p->t_model.get(); ba.t_mask = p->t_mask.get(); ba.t_action = p->t_action.get();
    ba.t_logp = p->t_logp.get(); ba.t_reward = p->t_reward.get(); ba.t_done = p->t_done.get();
    ba.obs = p->L.i_obs.get(); ba.model = p->L.i_model.get(); ba.mask = p->L.i_mask.get(); ba.action = p->L.i_action.get();
    ba.blogp = p->L.i_blogp.get(); ba.reward = p->L.i_reward.get(); ba.done = p->L.i_done.get(); ba.n_rows = p->L.i_n_rows.get();
    ramp_impala_batch_kernel<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(ba);
    CUDA_TRY(cudaGetLastError());
    // 2. one SGD step per train batch, in order
    AdamArgs aa = adam_args(p, *cfg, p->L.i_n_rows.get(), mb);
    aa.stats = p->L.i_stats.get();                                      // IMPALA's statistics: ramp_impala_step_stats_kernel
    for (int k = 0; k < n_sgd; ++k) {
        const int32_t start = k * mb, nf = std::min(F, n_frag - k * F);
        // the rounds at the current weights, kept for the backward; from the second step on also the embeddings, which the
        // previous update made stale (the first uses those the trajectory was collected with)
        if ((rc = launch_states(p, st, p->L.i_n_rows.get(), start, k ? p->d_emb.get() : nullptr)) != RAMP_OK) return rc;
        GradArgs ga{};
        ga.mb = mb; ga.start = start; ga.n_rows = p->L.i_n_rows.get();
        if ((rc = impala_batch(p, st, *cfg, L, start, nf, p->L.i_obs.get(), nullptr, p->L.i_model.get(), p->L.i_mask.get(), p->L.i_action.get(),
                               p->L.i_blogp.get(), p->L.i_reward.get(), p->L.i_done.get(), ga,
                               p->L.i_step_stats.get() + (size_t)k * RAMP_IMPALA_STATS_LEN)) != RAMP_OK)
            return rc;
        aa.start = start;
        if ((rc = launch_adam(p, aa, st)) != RAMP_OK) return rc;
    }
    p->emb_valid = false;
    p->L.i_rows = R;
    // 3. the means over the steps: the call's one read-back
    ramp_impala_learn_stats_kernel<<<1, 1, 0, st>>>(p->L.i_step_stats.get(), n_sgd, p->L.i_stats.get());
    CUDA_TRY(cudaGetLastError());
    ramp_internal_count_launches(eng, 2 + 9 * n_sgd);
    if (stats_out) CUDA_TRY(cudaMemcpyAsync(stats_out, p->L.i_stats.get(), sizeof(double) * RAMP_IMPALA_STATS_LEN, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

int ramp_impala_vtrace_read(ramp_policy_t* p, int32_t* n_out, float* target_logp_out, float* log_rho_out, float* vs_out,
                            float* pg_adv_out) {
    if (!p || !n_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (p->L.i_rows < 1) return set_error(RAMP_ERR_BAD_ARG, "impala: no V-trace yet (ramp_policy_learn_impala / ramp_impala_loss_grad)");
    CUDA_TRY(cudaSetDevice(p->device));
    CUDA_TRY(cudaDeviceSynchronize());
    const size_t n = (size_t)p->L.i_rows;
    *n_out = p->L.i_rows;
    if (target_logp_out) CUDA_TRY(cudaMemcpy(target_logp_out, p->L.i_tlogp.get(), 4 * n, cudaMemcpyDeviceToHost));
    if (log_rho_out) CUDA_TRY(cudaMemcpy(log_rho_out, p->L.i_log_rho.get(), 4 * n, cudaMemcpyDeviceToHost));
    if (vs_out) CUDA_TRY(cudaMemcpy(vs_out, p->L.i_vs.get(), 4 * n, cudaMemcpyDeviceToHost));
    if (pg_adv_out) CUDA_TRY(cudaMemcpy(pg_adv_out, p->L.i_pg.get(), 4 * n, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

// pg_torch_policy.py pg_torch_loss: -mean(logp(a) advantages) over the train batch, on host rows
int ramp_pg_loss_grad(ramp_policy_t* p, const ramp_pg_config_t* cfg, int32_t n, const int32_t* model, const float* graph_features,
                      const uint8_t* action_mask, const int32_t* action, const float* advantage, float* grad_out, double* stats_out) {
    if (!p || !model || !graph_features || !action_mask || !action || !advantage) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_learner_config(cfg);
    if (rc != RAMP_OK) return rc;
    if (n < 1) return set_error(RAMP_ERR_BAD_ARG, "pg: loss of %d rows", n);
    CUDA_TRY(cudaSetDevice(p->device));
    if ((rc = prepare_learner(p, 0, n)) ||
        (rc = upload_host_batch(p, n, model, graph_features, action_mask, nullptr, nullptr, action, nullptr, advantage, nullptr)))
        return rc;
    GradArgs ga = host_batch_args(p, n);
    ga.pg = 1; ga.action = p->h_action.get(); ga.adv = p->h_adv.get();
    if ((rc = launch_states(p, 0, nullptr, 0, nullptr)) != RAMP_OK || (rc = launch_grad(p, ga, 0)) != RAMP_OK) return rc;
    ramp_pg_stats_kernel<<<1, 1>>>(p->L.row_stats.get(), p->L.row_model.get(), p->h_adv.get(), n, ga.n_rows, p->L.norm_part.get(), p->L.stats.get());
    CUDA_TRY(cudaGetLastError());
    return host_batch_end(p, grad_out, stats_out, p->L.stats.get(), RAMP_PG_STATS_LEN);
}

// PG's training step (algorithms/pg: one learn_on_batch per train batch): post_process_advantages (compute_advantages with
// use_gae False, use_critic False, last_r 0), pg_torch_loss, torch.optim.Adam
int ramp_policy_learn_pg(ramp_policy_t* p, ramp_engine_t* eng, int32_t n_steps, const ramp_pg_config_t* cfg, double* stats_out) {
    ramp_env_buffers_t eb{};
    cudaStream_t st;
    int rc = learn_begin(p, eng, cfg, n_steps, "pg", &eb, &st);
    if (rc != RAMP_OK) return rc;
    const int32_t B = eb.n_episodes, rows = n_steps * B;
    if ((rc = prepare_learner(p, st, rows)) || (rc = ensure_batch(p->L, p->P.c, rows))) return rc;
    // 1. the discounted returns (ramp_ppo_gae_kernel without values: lambda 1, V = 0, a 0 bootstrap), the live rows t-major
    if ((rc = launch_gae(p, st, n_steps, B, cfg->gamma, 1.0, 0, nullptr)) != RAMP_OK) return rc;
    // 2. the loss's gradient over the whole batch at the collection weights (the embeddings the trajectory was collected with);
    //    the log p(a) the gradient kernel recomputes goes to b_logp_old
    GradArgs ga{};
    ga.mb = rows; ga.start = 0; ga.n_rows = p->L.n_rows.get(); ga.shuffle = 0; ga.obs_dyn = p->L.b_obs.get(); ga.model = p->L.b_model.get();
    ga.mask = p->L.b_mask.get(); ga.action = p->L.b_action.get(); ga.adv = p->L.b_adv.get(); ga.pg = 1; ga.logp_old = p->L.b_logp_old.get();
    if ((rc = launch_states(p, st, p->L.n_rows.get(), 0, nullptr)) != RAMP_OK || (rc = launch_grad(p, ga, st)) != RAMP_OK) return rc;
    // 3. one Adam step; with no row in the batch, none (the step count stays)
    AdamArgs aa = adam_args(p, *cfg, p->L.n_rows.get(), rows);
    aa.stats = p->L.stats.get();                                      // PG's statistics: ramp_pg_stats_kernel, after it
    if ((rc = launch_adam(p, aa, st)) != RAMP_OK) return rc;
    // 4. the statistics: the call's one read-back
    ramp_pg_stats_kernel<<<1, 1, 0, st>>>(p->L.row_stats.get(), p->L.row_model.get(), p->L.b_adv.get(), rows, p->L.n_rows.get(),
                                          p->L.norm_part.get(), p->L.stats.get());
    CUDA_TRY(cudaGetLastError());
    p->emb_valid = false;
    p->b_rows = rows;
    ramp_internal_count_launches(eng, 8);
    if (stats_out) CUDA_TRY(cudaMemcpyAsync(stats_out, p->L.stats.get(), sizeof(double) * RAMP_PG_STATS_LEN, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

}  // extern "C"

#include "ramp_population.cuh"
#include "ramp_es.cuh"
