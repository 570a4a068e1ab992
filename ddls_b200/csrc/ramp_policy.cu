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
//                           read-out (one hidden layer, logits; separate value branch), + max(log(mask), FLT_MIN) on the logits
//                           (gnn_policy.py:283-290), then greedy / categorical action selection written straight into the
//                           environment's action buffer.  All read-out weights are staged once per CTA in shared memory, laid
//                           out so that lanes read consecutive words.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
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

__global__ void __launch_bounds__(256) ramp_gnn_embed_kernel(const PolicyDev P, const ModelDev* models, float* emb) {
    __shared__ float sbuf[8][POL_MAX_DIM];
    const ModelDev M = models[blockIdx.x];
    if (M.n_nodes <= 0) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
    float* buf = sbuf[warp];
    const int half = P.c.out_features_msg / 2, msg = P.c.out_features_msg, akind = P.c.aggregator_activation;
    const float* zin = M.nf;
    int zin_stride = P.c.in_features_node;
    float* zout = M.z0;
    for (int r = 0; r < P.c.num_rounds; ++r) {
        const RoundW R = P.rounds[r];
        const float* w = P.w;
        // ---- node module on every node, edge module on every edge (mean_pool.py:120-127) ----
        for (int v = warp; v < M.n_nodes; v += n_warps) {
            for (int k = lane; k < R.in; k += 32) buf[k] = zin[(size_t)v * zin_stride + k];
            __syncwarp();
            warp_layer_norm(buf, R.in, w + R.nln_w, w + R.nln_b, lane);
            for (int o = lane; o < half; o += 32) {
                float a = w[R.nb + o];
                const float* row = w + R.nW + (size_t)o * R.in;
                for (int k = 0; k < R.in; ++k) a += row[k] * buf[k];
                M.hn[(size_t)v * half + o] = act_fn(a, akind);
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
                M.he[(size_t)e * half + o] = act_fn(a, akind);
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
            if (e1 > e0) {                                          // DGL leaves zero-in-degree nodes at zero
                for (int mi = -1; mi < e1 - e0; ++mi) {
                    const int src = mi < 0 ? v : M.in_src[e0 + mi];
                    for (int k = lane; k < half; k += 32) {
                        buf[k] = M.hn[(size_t)src * half + k];
                        buf[half + k] = mi < 0 ? 0.f : M.he[(size_t)M.in_edge[e0 + mi] * half + k];
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
                if (o < R.out) zout[(size_t)v * POL_MAX_DIM + o] = acc[i] * inv;
            }
        }
        __syncthreads();
        zin = zout; zin_stride = POL_MAX_DIM;
        zout = (zout == M.z0) ? M.z1 : M.z0;
    }
    // ---- mean over the job's nodes (gnn_policy.py:262-268) ----
    const int od = P.c.out_features_node;
    for (int o = threadIdx.x; o < od; o += blockDim.x) {
        float s = 0.f;
        for (int v = 0; v < M.n_nodes; ++v) s += zin[(size_t)v * POL_MAX_DIM + o];
        emb[(size_t)blockIdx.x * od + o] = s / (float)M.n_nodes;
    }
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
    const int gin = c.in_features_graph + c.n_actions, fin = c.out_features_node + c.out_features_graph, H = c.fcnet_hidden, A = c.n_actions;
    return (size_t)2 * gin + (size_t)c.out_features_graph * gin + c.out_features_graph      // graph module
           + (size_t)2 * fin * H + 2 * (size_t)H                                           // hidden layers (policy, value), transposed
           + (size_t)A * H + A + H + 1                                                      // logits, value
           + (size_t)warps * 2 * POL_MAX_DIM;                                               // per-warp staging
}

__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

__global__ void __launch_bounds__(256) ramp_policy_head_kernel(const PolicyDev P, const HeadArgs a) {
    extern __shared__ float sm[];
    const ramp_policy_config_t& c = P.c;
    const int gin = c.in_features_graph + c.n_actions, og = c.out_features_graph, on = c.out_features_node, fin = on + og;
    const int H = c.fcnet_hidden, A = c.n_actions, hpl = H / 32;
    float* s_gln_w = sm;                 float* s_gln_b = s_gln_w + gin;
    float* s_gW = s_gln_b + gin;         float* s_gb = s_gW + (size_t)og * gin;
    float* s_hWt = s_gb + og;            float* s_hb = s_hWt + (size_t)fin * H;      // [fin][H]: lanes read consecutive hidden units
    float* s_vhWt = s_hb + H;            float* s_vhb = s_vhWt + (size_t)fin * H;
    float* s_lW = s_vhb + H;             float* s_lb = s_lW + (size_t)A * H;         // [A][H]
    float* s_vW = s_lb + A;              float* s_vb = s_vW + H;
    float* s_warp = s_vb + 1;
    const float* w = P.w;
    for (int i = threadIdx.x; i < gin; i += blockDim.x) { s_gln_w[i] = w[P.gln_w + i]; s_gln_b[i] = w[P.gln_b + i]; }
    for (int i = threadIdx.x; i < og * gin; i += blockDim.x) s_gW[i] = w[P.gW + i];
    for (int i = threadIdx.x; i < og; i += blockDim.x) s_gb[i] = w[P.gb + i];
    for (int i = threadIdx.x; i < fin * H; i += blockDim.x) {
        const int j = i / fin, k = i - j * fin;                       // blob is [H][fin]
        s_hWt[(size_t)k * H + j] = w[P.hW + i];
        s_vhWt[(size_t)k * H + j] = w[P.vhW + i];
    }
    for (int i = threadIdx.x; i < H; i += blockDim.x) { s_hb[i] = w[P.hb + i]; s_vhb[i] = w[P.vhb + i]; s_vW[i] = w[P.vW + i]; }
    for (int i = threadIdx.x; i < A * H; i += blockDim.x) s_lW[i] = w[P.lW + i];
    for (int i = threadIdx.x; i < A; i += blockDim.x) s_lb[i] = w[P.lb + i];
    if (threadIdx.x == 0) s_vb[0] = w[P.vb];
    __syncthreads();

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wpc = blockDim.x >> 5;
    float* xb = s_warp + (size_t)warp * 2 * POL_MAX_DIM;                // graph-module input, then the read-out input
    float* fb = xb + POL_MAX_DIM;
    for (int b = blockIdx.x * wpc + warp; b < a.n; b += gridDim.x * wpc) {
        const int m = a.model[b];
        const bool live = m >= 0 && m < c.n_models && !(a.done && a.done[b]);
        if (!live) {                                                    // nothing queued: the action is ignored by the environment
            if (lane < A && a.logits) a.logits[(size_t)b * A + lane] = 0.f;
            if (lane == 0) { a.actions[b] = 0; if (a.value) a.value[b] = 0.f; if (a.logp) a.logp[b] = 0.f; }
            continue;
        }
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
        warp_layer_norm(xb, gin, s_gln_w, s_gln_b, lane);
        for (int k = lane; k < on; k += 32) fb[k] = a.emb[(size_t)m * on + k];
        if (lane < og) {
            float g = s_gb[lane];
            const float* row = s_gW + (size_t)lane * gin;
            for (int k = 0; k < gin; ++k) g += row[k] * xb[k];
            fb[on + lane] = g;
        }
        __syncwarp();
        // ---- read-out: hidden layer of the policy and of the value branch, each lane owns units lane + 32 i ----
        float h[POL_MAX_HPL], hv[POL_MAX_HPL];
#pragma unroll
        for (int i = 0; i < POL_MAX_HPL; ++i) {
            if (i < hpl) {
                const int j = lane + 32 * i;
                float p = s_hb[j], q = s_vhb[j];
                for (int k = 0; k < fin; ++k) { const float f = fb[k]; p += s_hWt[(size_t)k * H + j] * f; q += s_vhWt[(size_t)k * H + j] * f; }
                h[i] = act_fn(p, c.fcnet_activation); hv[i] = act_fn(q, c.fcnet_activation);
            }
        }
        float my_logit = -FLT_MAX;
        for (int o = 0; o < A; ++o) {
            float p = 0.f;
#pragma unroll
            for (int i = 0; i < POL_MAX_HPL; ++i) if (i < hpl) p += h[i] * s_lW[(size_t)o * H + lane + 32 * i];
            p = warp_sum(p) + s_lb[o];
            if (c.apply_action_mask && !a.mask[(size_t)b * A + o]) p += -FLT_MAX;   // + max(log 0, finfo.min) (gnn_policy.py:285-290)
            if (lane == o) my_logit = p;
        }
        float val = 0.f;
#pragma unroll
        for (int i = 0; i < POL_MAX_HPL; ++i) if (i < hpl) val += hv[i] * s_vW[lane + 32 * i];
        val = warp_sum(val) + s_vb[0];
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
    unsigned long long act_calls = 0;
    // trajectory of a rollout segment (ramp_policy_trajectory_*): [horizon][B] per field, on the device until read
    int32_t traj_h = 0, traj_b = 0, traj_a = 0;
    int32_t traj_n = 0;                   // slots recorded in order, both phases, since ramp_policy_trajectory_begin
    DeviceArray<float> t_obs, t_logp, t_value; DeviceArray<int32_t> t_model, t_action;
    DeviceArray<uint8_t> t_mask, t_done; DeviceArray<double> t_reward;
    // learner (ramp_policy_backward / ramp_ppo_loss_grad / ramp_policy_learn): gradient, Adam's moments and step count, per job type
    // gradients, norm partials; per-row scratch for `lcap` rows, the head segments for `seg_n` rows
    bool learner_ready = false, gmodels_ready = false;
    int32_t adam_parity = 0, lcap = 0, seg_n = 0;
    int64_t seg_total = 0;
    DeviceArray<float> l_grad, l_adam_m, l_adam_v, l_gpart, l_rec, l_row_stats;
    DeviceArray<int32_t> l_n_rows, l_step, l_row_model;
    DeviceArray<double> l_norm_part, l_stats, l_mb_stats;
    DeviceArray<Seg> l_segs;
    DeviceArray<GradModelDev> d_gmodels;
    // host-input batches of ramp_policy_backward / ramp_ppo_loss_grad
    int32_t hcap = 0;
    DeviceArray<int32_t> h_model, h_action; DeviceArray<float> h_gf, h_gl, h_gv, h_old, h_adv, h_vt; DeviceArray<uint8_t> h_mask;
    // ramp_policy_learn's / ramp_policy_learn_pg's train batch ([horizon * B] rows, live rows first, t-major) and bootstrap values ([B])
    int32_t bcap = 0, boot_cap = 0, b_rows = 0;
    DeviceArray<float> b_obs, b_logp, b_logp_old, b_adv, b_vt, b_old, b_value, b_lpx, l_boot;
    DeviceArray<int32_t> b_model, b_action, b_actx, l_boot_act; DeviceArray<uint8_t> b_mask; DeviceArray<double> b_adv64;
    // IMPALA (ramp_policy_learn_impala / ramp_impala_loss_grad): the fragment rows ([icap], row f L + t) with their read-out at
    // the current weights and V-trace values, the loss's job types (-1 outside it), the host batch's extra inputs, statistics
    int32_t icap = 0, i_rows = 0, i_step_cap = 0;
    DeviceArray<float> i_obs, i_blogp, i_tlogits, i_tvalue, i_tlogp, i_log_rho, i_vs, i_pg;
    DeviceArray<int32_t> i_model, i_action, i_actx, i_lmodel, i_n_rows; DeviceArray<uint8_t> i_mask, i_done;
    DeviceArray<double> i_reward, i_step_stats, i_stats;
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
    const int64_t vhW = take((int64_t)H * fin), vhb = take(H), vW = take(H), vb = take(1);
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
    if (c.fcnet_hidden < 32 || c.fcnet_hidden % 32 || c.fcnet_hidden > 32 * POL_MAX_HPL)
        return set_error(RAMP_ERR_BAD_ARG, "policy: fcnet_hidden must be a multiple of 32 in [32, %d]", 32 * POL_MAX_HPL);
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

int launch_embed(ramp_policy* p, cudaStream_t st) {
    for (size_t m = 0; m < p->models.size(); ++m)
        if (!p->models[m].set) return set_error(RAMP_ERR_BAD_ARG, "policy: model %zu was never registered (ramp_policy_set_model)", m);
    if (!p->weights_set) return set_error(RAMP_ERR_BAD_ARG, "policy: no weights (ramp_policy_set_weights)");
    std::vector<ModelDev> h(p->models.size());
    for (size_t m = 0; m < h.size(); ++m) h[m] = p->models[m].d;
    CUDA_TRY(cudaMemcpyAsync(p->d_models.get(), h.data(), sizeof(ModelDev) * h.size(), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));                                  // `h` is pageable
    ramp_gnn_embed_kernel<<<(unsigned)h.size(), 256, 0, st>>>(p->P, p->d_models.get(), p->d_emb.get());
    CUDA_TRY(cudaGetLastError());
    p->emb_valid = true;
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

// the read-out on host inputs (ramp_policy_forward / ramp_policy_decide), in buffers of its own: what the last act left for
// ramp_policy_read and the trajectory stays as it was
int head_on_host(ramp_policy* p, int32_t n, const int32_t* model, const float* graph_features, const uint8_t* action_mask, int32_t sample,
                 uint64_t seed, float* logits_out, float* value_out, float* logp_out, int32_t* actions_out) {
    if (!p || !model || !graph_features || !action_mask) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n < 1) return RAMP_OK;
    const ramp_policy_config_t& c = p->P.c;
    CUDA_TRY(cudaSetDevice(p->device));
    int rc;
    if (!p->emb_valid && (rc = launch_embed(p, 0)) != RAMP_OK) return rc;
    if (n > p->fcap) {
        p->fcap = 0;                      // until every buffer has the new size
        CUDA_TRY(alloc_each(n, p->f_model, p->f_actions, p->f_value, p->f_logp));
        CUDA_TRY(p->f_gf.alloc((size_t)n * c.in_features_graph));
        CUDA_TRY(alloc_each((size_t)n * c.n_actions, p->f_mask, p->f_logits));
        p->fcap = n;
    }
    CUDA_TRY(cudaMemcpy(p->f_model.get(), model, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(p->f_gf.get(), graph_features, sizeof(float) * (size_t)n * c.in_features_graph, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(p->f_mask.get(), action_mask, (size_t)n * c.n_actions, cudaMemcpyHostToDevice));
    HeadArgs a{};
    a.n = n; a.graph_features = p->f_gf.get(); a.model = p->f_model.get(); a.mask = p->f_mask.get(); a.emb = p->d_emb.get(); a.graph_static = p->d_gstatic.get();
    a.logits = p->f_logits.get(); a.value = p->f_value.get(); a.logp = p->f_logp.get(); a.actions = p->f_actions.get();
    a.sample = sample; a.seed = seed;
    if ((rc = launch_head(p, a, 0)) != RAMP_OK) return rc;
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

int ensure_learner(ramp_policy* p) {
    if (p->learner_ready) return RAMP_OK;
    const size_t nw = (size_t)p->n_weights;
    CUDA_TRY(alloc_each(nw, p->l_grad, p->l_adam_m, p->l_adam_v));
    CUDA_TRY(p->l_gpart.alloc((size_t)p->P.c.n_models * gnn_weight_count(p)));
    CUDA_TRY(p->l_n_rows.alloc(2));                                  // [0] learn's train batch, [1] a host batch
    CUDA_TRY(p->l_step.alloc(2));
    CUDA_TRY(p->l_norm_part.alloc(LRN_GRID));
    CUDA_TRY(p->l_stats.alloc(RAMP_PPO_STATS_LEN));
    CUDA_TRY(p->l_segs.alloc(HEAD_SEGS));
    CUDA_TRY(p->d_gmodels.alloc(p->P.c.n_models));
    CUDA_TRY(cudaMemset(p->l_adam_m.get(), 0, sizeof(float) * nw));
    CUDA_TRY(cudaMemset(p->l_adam_v.get(), 0, sizeof(float) * nw));
    CUDA_TRY(cudaMemset(p->l_step.get(), 0, sizeof(int32_t) * 2));
    p->adam_parity = 0;
    p->learner_ready = true;
    return RAMP_OK;
}

// every job type's forward states and records for the embedding backward, sized by its graph
int ensure_gmodels(ramp_policy* p) {
    if (p->gmodels_ready) return RAMP_OK;
    const ramp_policy_config_t& c = p->P.c;
    const GnnDims D = gnn_dims(c);
    const size_t half = c.out_features_msg / 2, R = c.num_rounds;
    std::vector<GradModelDev> h(p->models.size());
    for (size_t m = 0; m < h.size(); ++m) {
        HostModel& hm = p->models[m];
        if (!hm.set) return set_error(RAMP_ERR_BAD_ARG, "policy: model %zu was never registered (ramp_policy_set_model)", m);
        if (!hm.grad_ready) {
            hm.lallocs.clear();
            const size_t N = hm.d.n_nodes, E = hm.d.n_edges;
            auto take = [&](size_t floats, float** dst) -> int {
                hm.lallocs.emplace_back();
                CUDA_TRY(hm.lallocs.back().alloc(sizeof(float) * floats));
                *dst = (float*)hm.lallocs.back().get();
                return RAMP_OK;
            };
            GradModelDev& g = hm.g;
            int rc;
            if ((rc = take(R * N * D.zs, &g.z)) || (rc = take(R * N * half, &g.hn)) || (rc = take(R * E * half, &g.he)) ||
                (rc = take(N * D.zs, &g.dz)) || (rc = take(N * D.zs, &g.dz2)) || (rc = take(N * half, &g.dhn)) ||
                (rc = take(N * D.nrs, &g.nrec)) || (rc = take(E * D.ers, &g.erec)) || (rc = take((N + E) * D.mrs, &g.mrec)) ||
                (rc = take((N + E) * c.out_features_msg, &g.mdx)))
                return rc;
            hm.grad_ready = true;
        }
        h[m] = hm.g;
    }
    CUDA_TRY(cudaMemcpy(p->d_gmodels.get(), h.data(), sizeof(GradModelDev) * h.size(), cudaMemcpyHostToDevice));
    p->gmodels_ready = true;
    return RAMP_OK;
}

// per-row scratch for minibatches of n rows, and the head segments summing exactly n rows
int ensure_rows(ramp_policy* p, int32_t n) {
    if (n > p->lcap) {
        p->lcap = 0;
        p->seg_n = 0;
        CUDA_TRY(p->l_rec.alloc((size_t)n * head_rec(p->P.c).stride));
        CUDA_TRY(p->l_row_stats.alloc((size_t)n * RS_N));
        CUDA_TRY(p->l_row_model.alloc(n));
        p->lcap = n;
    }
    if (n != p->seg_n) {
        Seg s[HEAD_SEGS];
        head_segs(p->P, p->l_rec.get(), n, s);
        p->seg_total = 0;
        for (const Seg& x : s) p->seg_total += seg_size(x);
        CUDA_TRY(cudaMemcpy(p->l_segs.get(), s, sizeof(s), cudaMemcpyHostToDevice));
        p->seg_n = n;
    }
    return RAMP_OK;
}

int prepare_learner(ramp_policy* p, cudaStream_t st) {
    int rc;
    if ((rc = ensure_learner(p)) != RAMP_OK || (rc = ensure_gmodels(p)) != RAMP_OK) return rc;
    if (!p->emb_valid && (rc = launch_embed(p, st)) != RAMP_OK) return rc;
    return RAMP_OK;
}

// the MeanPool rounds of every job type, kept for the backward (and the embeddings when `emb` is given); nothing for a minibatch
// starting at `start` past the end of a batch of *n_rows rows (n_rows may be nullptr)
int launch_states(ramp_policy* p, cudaStream_t st, const int32_t* n_rows, int32_t start, float* emb) {
    EmbGradArgs eg{};
    eg.n_rows = n_rows; eg.start = start; eg.emb = emb;
    ramp_gnn_embed_grad_kernel<EMB_FORWARD><<<p->P.c.n_models, 256, 0, st>>>(p->P, p->d_models.get(), p->d_gmodels.get(), eg);
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

// head gradient -> head reduction -> embedding gradient (from launch_states' states) -> per-job-type sum and norm partials:
// the gradient in l_grad
int launch_grad(ramp_policy* p, GradArgs ga, cudaStream_t st) {
    ga.rec = p->l_rec.get(); ga.row_model = p->l_row_model.get(); ga.row_stats = p->l_row_stats.get();
    ga.emb = p->d_emb.get(); ga.graph_static = p->d_gstatic.get();
    ramp_policy_head_grad_kernel<<<(ga.mb + LRN_WARPS - 1) / LRN_WARPS, LRN_WARPS * 32, 0, st>>>(p->P, ga);
    int64_t grid = (p->seg_total + 255) / 256;
    if (grid > 4 * p->sm_count) grid = 4 * p->sm_count;
    ramp_policy_head_reduce_kernel<<<(unsigned)grid, 256, 0, st>>>(p->P, p->l_segs.get(), HEAD_SEGS, p->seg_total, p->l_grad.get());
    EmbGradArgs eg{};
    eg.rec = p->l_rec.get(); eg.row_model = p->l_row_model.get(); eg.rows = ga.mb; eg.gpart = p->l_gpart.get(); eg.n_gnn = gnn_weight_count(p);
    ramp_gnn_embed_grad_kernel<EMB_BACKWARD><<<p->P.c.n_models, 256, 0, st>>>(p->P, p->d_models.get(), p->d_gmodels.get(), eg);
    ramp_grad_finish_kernel<<<LRN_GRID, 256, 0, st>>>(p->l_gpart.get(), p->P.c.n_models, gnn_weight_count(p), p->n_weights,
                                                       p->l_grad.get(), p->l_norm_part.get());
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

int check_ppo_config(const ramp_ppo_config_t* cfg) {
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

// the host inputs of ramp_policy_backward / ramp_ppo_loss_grad on the device (any pointer may be NULL: not copied)
int upload_host_batch(ramp_policy* p, int32_t n, const int32_t* model, const float* gf, const uint8_t* mask, const float* gl,
                      const float* gv, const int32_t* action, const float* old_logits, const float* adv, const float* vt) {
    const ramp_policy_config_t& c = p->P.c;
    const size_t A = c.n_actions;
    if (n > p->hcap) {
        p->hcap = 0;
        CUDA_TRY(alloc_each(n, p->h_model, p->h_action, p->h_gv, p->h_adv, p->h_vt));
        CUDA_TRY(p->h_gf.alloc((size_t)n * c.in_features_graph));
        CUDA_TRY(alloc_each((size_t)n * A, p->h_gl, p->h_old, p->h_mask));
        p->hcap = n;
    }
    auto put = [&](void* dst, const void* src, size_t bytes) -> int {
        if (src) CUDA_TRY(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice));
        return RAMP_OK;
    };
    int rc;
    if ((rc = put(p->h_model.get(), model, 4 * (size_t)n)) || (rc = put(p->h_gf.get(), gf, 4 * (size_t)n * c.in_features_graph)) ||
        (rc = put(p->h_mask.get(), mask, (size_t)n * A)) || (rc = put(p->h_gl.get(), gl, 4 * (size_t)n * A)) ||
        (rc = put(p->h_gv.get(), gv, 4 * (size_t)n)) || (rc = put(p->h_action.get(), action, 4 * (size_t)n)) ||
        (rc = put(p->h_old.get(), old_logits, 4 * (size_t)n * A)) || (rc = put(p->h_adv.get(), adv, 4 * (size_t)n)) ||
        (rc = put(p->h_vt.get(), vt, 4 * (size_t)n)) || (rc = put(p->l_n_rows.get() + 1, &n, 4)))
        return rc;
    for (int32_t b = 0; b < n; ++b)
        if (action && model[b] >= 0 && model[b] < c.n_models && (action[b] < 0 || action[b] >= c.n_actions))
            return set_error(RAMP_ERR_BAD_ARG, "ppo: action %d of row %d outside [0, %d)", action[b], b, c.n_actions);
    return RAMP_OK;
}

// the train batch of ramp_policy_learn / ramp_policy_learn_pg for `rows` trajectory slots
int ensure_batch(ramp_policy* p, int32_t rows) {
    if (rows <= p->bcap) return RAMP_OK;
    p->bcap = 0;
    CUDA_TRY(alloc_each(rows, p->b_logp, p->b_logp_old, p->b_adv, p->b_vt, p->b_value, p->b_lpx, p->b_model, p->b_action, p->b_actx, p->b_adv64));
    CUDA_TRY(p->b_obs.alloc((size_t)rows * 11));
    CUDA_TRY(alloc_each((size_t)rows * p->P.c.n_actions, p->b_mask, p->b_old));
    p->bcap = rows;
    return RAMP_OK;
}

GradArgs host_batch_args(ramp_policy* p, int32_t n) {
    GradArgs ga{};
    ga.mb = n; ga.start = 0; ga.n_rows = p->l_n_rows.get() + 1;
    ga.graph_features = p->h_gf.get(); ga.model = p->h_model.get(); ga.mask = p->h_mask.get();
    return ga;
}

int check_impala_config(const ramp_impala_config_t* cfg) {
    if (!cfg) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (!(cfg->vtrace_clip_rho_threshold > 0) || !(cfg->vtrace_clip_pg_rho_threshold > 0) || !(cfg->lr >= 0) || !(cfg->adam_eps > 0))
        return set_error(RAMP_ERR_BAD_ARG, "impala: the clip thresholds and adam_eps must be > 0, lr >= 0");
    if (cfg->rollout_fragment_length < 0 || cfg->train_batch_size < 1)
        return set_error(RAMP_ERR_BAD_ARG, "impala: rollout_fragment_length must be >= 0, train_batch_size >= 1");
    return RAMP_OK;
}

int check_pg_config(const ramp_pg_config_t* cfg) {
    if (!cfg) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (!(cfg->gamma >= 0) || !(cfg->lr >= 0) || !(cfg->adam_eps > 0)) return set_error(RAMP_ERR_BAD_ARG, "pg: gamma and lr must be >= 0, adam_eps > 0");
    return RAMP_OK;
}

// IMPALA's per-row arrays for n fragment rows, and statistics for `steps` SGD steps
int ensure_impala(ramp_policy* p, int32_t n, int32_t steps) {
    const size_t A = p->P.c.n_actions;
    if (n > p->icap) {
        p->icap = 0;
        CUDA_TRY(alloc_each(n, p->i_blogp, p->i_tvalue, p->i_tlogp, p->i_log_rho, p->i_vs, p->i_pg, p->i_model, p->i_action,
                            p->i_actx, p->i_lmodel, p->i_done, p->i_reward));
        CUDA_TRY(p->i_obs.alloc((size_t)n * 11));
        CUDA_TRY(alloc_each((size_t)n * A, p->i_tlogits, p->i_mask));
        p->icap = n;
    }
    if (!p->i_n_rows.get()) {
        CUDA_TRY(p->i_n_rows.alloc(1));
        CUDA_TRY(p->i_stats.alloc(RAMP_IMPALA_STATS_LEN));
    }
    if (steps > p->i_step_cap) {
        p->i_step_cap = 0;
        CUDA_TRY(p->i_step_stats.alloc((size_t)steps * RAMP_IMPALA_STATS_LEN));
        p->i_step_cap = steps;
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
    h.logits = p->i_tlogits.get() + r0 * A; h.value = p->i_tvalue.get() + r0; h.actions = p->i_actx.get() + r0;
    if ((rc = launch_head(p, h, st)) != RAMP_OK) return rc;
    VtraceArgs v{};
    v.L = L; v.n_frag = n_frag; v.row0 = row0; v.A = c.n_actions; v.n_models = c.n_models;
    v.gamma = cfg.gamma; v.clip_rho = cfg.vtrace_clip_rho_threshold; v.clip_pg_rho = cfg.vtrace_clip_pg_rho_threshold;
    v.logits = p->i_tlogits.get(); v.value = p->i_tvalue.get();
    v.model = model; v.action = action; v.blogp = blogp; v.reward = reward; v.done = done;
    v.tlogp = p->i_tlogp.get(); v.log_rho = p->i_log_rho.get(); v.vs = p->i_vs.get(); v.pg_adv = p->i_pg.get(); v.lmodel = p->i_lmodel.get();
    ramp_vtrace_kernel<<<(unsigned)((n_frag + 7) / 8), 256, 0, st>>>(v);
    CUDA_TRY(cudaGetLastError());
    ga.impala = 1; ga.shuffle = 0; ga.graph_features = graph_features; ga.obs_dyn = obs_dyn; ga.model = p->i_lmodel.get(); ga.mask = mask;
    ga.action = action; ga.adv = p->i_pg.get(); ga.vt = p->i_vs.get();
    ga.vf_coeff = (float)cfg.vf_loss_coeff; ga.ent_coeff = (float)cfg.entropy_coeff;
    if ((rc = launch_grad(p, ga, st)) != RAMP_OK) return rc;
    ramp_impala_step_stats_kernel<<<1, 1, 0, st>>>(p->l_row_stats.get(), p->l_row_model.get(), ga.mb, row0, p->i_log_rho.get(),
                                                   cfg.vf_loss_coeff, cfg.entropy_coeff, p->l_norm_part.get(), stats);
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
    hm.set = hm.grad_ready = p->gmodels_ready = false;
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
    hm.set = true;
    p->emb_valid = false;
    return RAMP_OK;
}

int ramp_policy_embed(ramp_policy_t* p, float* embeddings_out) {
    if (!p) return set_error(RAMP_ERR_BAD_ARG, "null policy");
    CUDA_TRY(cudaSetDevice(p->device));
    int rc = launch_embed(p, 0);
    if (rc != RAMP_OK) return rc;
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
    if (!p->emb_valid) { if ((rc = launch_embed(p, st)) != RAMP_OK) return rc; ++launches; }
    if ((rc = ensure_outputs(p, eb.n_episodes)) != RAMP_OK) return rc;
    HeadArgs a{};
    a.n = eb.n_episodes; a.obs_dyn = eb.obs_dynamic; a.graph_static = p->d_gstatic.get(); a.model = eb.queued_model; a.done = eb.done;
    a.mask = eb.action_mask; a.emb = p->d_emb.get(); a.logits = p->d_logits.get(); a.value = p->d_value.get(); a.logp = p->d_logp.get(); a.actions = eb.actions;
    a.sample = sample; a.seed = seed ^ (0x9E3779B97F4A7C15ull * (++p->act_calls));
    if ((rc = launch_head(p, a, st)) != RAMP_OK) return rc;
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
    if ((rc = prepare_learner(p, 0)) || (rc = ensure_rows(p, n)) ||
        (rc = upload_host_batch(p, n, model, graph_features, action_mask, grad_logits, grad_value, nullptr, nullptr, nullptr, nullptr)))
        return rc;
    GradArgs ga = host_batch_args(p, n);
    ga.grad_logits = p->h_gl.get(); ga.grad_value = p->h_gv.get();
    if ((rc = launch_states(p, 0, nullptr, 0, nullptr)) != RAMP_OK || (rc = launch_grad(p, ga, 0)) != RAMP_OK) return rc;
    CUDA_TRY(cudaStreamSynchronize(0));
    CUDA_TRY(cudaMemcpy(grad_weights_out, p->l_grad.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_ppo_loss_grad(ramp_policy_t* p, const ramp_ppo_config_t* cfg, int32_t n, const int32_t* model, const float* graph_features,
                       const uint8_t* action_mask, const int32_t* action, const float* old_logits, const float* advantage,
                       const float* value_target, float* grad_out, double* stats_out) {
    if (!p || !model || !graph_features || !action_mask || !action || !old_logits || !advantage || !value_target)
        return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_ppo_config(cfg);
    if (rc != RAMP_OK) return rc;
    if (n < 1) return set_error(RAMP_ERR_BAD_ARG, "ppo: loss of %d rows", n);
    CUDA_TRY(cudaSetDevice(p->device));
    if ((rc = prepare_learner(p, 0)) || (rc = ensure_rows(p, n)) ||
        (rc = upload_host_batch(p, n, model, graph_features, action_mask, nullptr, nullptr, action, old_logits, advantage, value_target)))
        return rc;
    GradArgs ga = host_batch_args(p, n);
    ga.action = p->h_action.get(); ga.old_logits = p->h_old.get(); ga.adv = p->h_adv.get(); ga.vt = p->h_vt.get();
    ppo_terms(ga, *cfg);
    if ((rc = launch_states(p, 0, nullptr, 0, nullptr)) != RAMP_OK || (rc = launch_grad(p, ga, 0)) != RAMP_OK) return rc;
    ramp_ppo_minibatch_stats_kernel<<<1, 1>>>(p->l_row_stats.get(), n, ga.vf_coeff, ga.ent_coeff, ga.kl_coeff, p->l_norm_part.get(), p->l_stats.get());
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(0));
    if (grad_out) CUDA_TRY(cudaMemcpy(grad_out, p->l_grad.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToHost));
    if (stats_out) CUDA_TRY(cudaMemcpy(stats_out, p->l_stats.get(), sizeof(double) * RAMP_PPO_STATS_LEN, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_policy_learn(ramp_policy_t* p, ramp_engine_t* eng, int32_t n_steps, const ramp_ppo_config_t* cfg, double* stats_out) {
    if (!p || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_ppo_config(cfg);
    if (rc != RAMP_OK) return rc;
    ramp_env_buffers_t eb{};
    if ((rc = ramp_env_buffers(eng, &eb)) != RAMP_OK) return rc;
    if (n_steps < 1 || n_steps > p->traj_n)
        return set_error(RAMP_ERR_BAD_ARG, "ppo: %d steps asked of a trajectory with %d recorded", n_steps, p->traj_n);
    if (eb.n_episodes != p->traj_b || eb.n_actions != p->traj_a)
        return set_error(RAMP_ERR_BAD_ARG, "ppo: the trajectory was recorded from another environment");
    const ramp_policy_config_t& c = p->P.c;
    CUDA_TRY(cudaSetDevice(p->device));
    cudaStream_t st = ramp_internal_stream(eng);
    const int32_t B = eb.n_episodes, rows = n_steps * B, mb = cfg->sgd_minibatch_size, n_mb = (rows + mb - 1) / mb;
    if ((rc = prepare_learner(p, st)) || (rc = ensure_rows(p, mb)) || (rc = ensure_batch(p, rows))) return rc;
    if (B > p->boot_cap) {
        p->boot_cap = 0;
        CUDA_TRY(alloc_each(B, p->l_boot, p->l_boot_act));
        p->boot_cap = B;
    }
    if ((size_t)n_mb * RAMP_PPO_STATS_LEN > p->l_mb_stats.size()) CUDA_TRY(p->l_mb_stats.alloc((size_t)n_mb * RAMP_PPO_STATS_LEN));
    int launches = 2;                                                   // GAE, old logits
    // 1. the value of the state after the last step (RLlib's truncate_episodes bootstrap): when the trajectory goes on, the value
    //    act recorded in slot n_steps; after its last recorded slot, the environment's current state, by the head kernel on its
    //    buffers -- not through ramp_policy_act, which mixes its call count into the seed and writes the action buffer
    const float* boot = p->t_value.get() + (size_t)n_steps * B;
    if (n_steps == p->traj_n) {
        HeadArgs hb{};
        hb.n = B; hb.obs_dyn = eb.obs_dynamic; hb.graph_static = p->d_gstatic.get(); hb.model = eb.queued_model; hb.done = eb.done;
        hb.mask = eb.action_mask; hb.emb = p->d_emb.get(); hb.value = p->l_boot.get(); hb.actions = p->l_boot_act.get();
        if ((rc = launch_head(p, hb, st)) != RAMP_OK) return rc;
        boot = p->l_boot.get();
        ++launches;
    }
    // 2. GAE, the live rows t-major, standardised advantages
    GaeArgs ge{};
    ge.T = n_steps; ge.B = B; ge.A = c.n_actions; ge.n_models = c.n_models; ge.standardize = cfg->standardize_advantages;
    ge.gamma = cfg->gamma; ge.lambda = cfg->lambda;
    ge.t_obs = p->t_obs.get(); ge.t_model = p->t_model.get(); ge.t_mask = p->t_mask.get(); ge.t_action = p->t_action.get();
    ge.t_logp = p->t_logp.get(); ge.t_value = p->t_value.get(); ge.t_reward = p->t_reward.get(); ge.t_done = p->t_done.get();
    ge.boot = boot; ge.adv64 = p->b_adv64.get();
    ge.obs = p->b_obs.get(); ge.model = p->b_model.get(); ge.mask = p->b_mask.get(); ge.action = p->b_action.get(); ge.logp = p->b_logp.get();
    ge.adv = p->b_adv.get(); ge.vt = p->b_vt.get(); ge.n_rows = p->l_n_rows.get();
    ramp_ppo_gae_kernel<<<1, 1024, 0, st>>>(ge);
    CUDA_TRY(cudaGetLastError());
    // 3. the collection weights' logits of every row: the head kernel again, so they are act's bits
    HeadArgs ho{};
    ho.n = rows; ho.obs_dyn = p->b_obs.get(); ho.graph_static = p->d_gstatic.get(); ho.model = p->b_model.get(); ho.mask = p->b_mask.get();
    ho.emb = p->d_emb.get(); ho.logits = p->b_old.get(); ho.value = p->b_value.get(); ho.logp = p->b_lpx.get(); ho.actions = p->b_actx.get();
    if ((rc = launch_head(p, ho, st)) != RAMP_OK) return rc;
    // 4. num_sgd_iter shuffled passes of minibatch updates; a minibatch past the batch's end (its size is on the device) is a no-op
    GradArgs ga{};
    ga.mb = mb; ga.n_rows = p->l_n_rows.get(); ga.shuffle = 1; ga.obs_dyn = p->b_obs.get(); ga.model = p->b_model.get();
    ga.mask = p->b_mask.get(); ga.action = p->b_action.get(); ga.old_logits = p->b_old.get(); ga.adv = p->b_adv.get(); ga.vt = p->b_vt.get();
    ppo_terms(ga, *cfg);
    AdamArgs aa{};
    aa.lr = cfg->lr; aa.beta1 = cfg->adam_beta1; aa.beta2 = cfg->adam_beta2;
    aa.beta2_f = (float)cfg->adam_beta2; aa.one_m_beta1 = (float)(1.0 - cfg->adam_beta1); aa.one_m_beta2 = (float)(1.0 - cfg->adam_beta2);
    aa.eps = (float)cfg->adam_eps;
    aa.max_norm = (float)cfg->grad_clip; aa.n_rows = p->l_n_rows.get(); aa.mb = mb; aa.step = p->l_step.get();
    aa.m = p->l_adam_m.get(); aa.v = p->l_adam_v.get(); aa.grad = p->l_grad.get(); aa.norm_part = p->l_norm_part.get(); aa.w = p->d_w.get();
    aa.row_stats = p->l_row_stats.get(); aa.vf_coeff = ga.vf_coeff; aa.ent_coeff = ga.ent_coeff; aa.kl_coeff = ga.kl_coeff;
    for (int pass = 0; pass < cfg->num_sgd_iter; ++pass) {
        ga.key = mix64(cfg->seed ^ mix64((uint64_t)pass + 1));
        ga.logp_old = pass == 0 ? p->b_logp_old.get() : nullptr;
        for (int k = 0; k < n_mb; ++k) {
            // the rounds at the current weights, kept for the backward; from the second minibatch on also the embeddings, which
            // the previous update made stale (the first uses those the old logits were computed with)
            ga.start = aa.start = k * mb;
            if ((rc = launch_states(p, st, p->l_n_rows.get(), ga.start, pass || k ? p->d_emb.get() : nullptr)) != RAMP_OK ||
                (rc = launch_grad(p, ga, st)) != RAMP_OK)
                return rc;
            aa.parity = p->adam_parity; p->adam_parity ^= 1;
            aa.stats = p->l_mb_stats.get() + (size_t)k * RAMP_PPO_STATS_LEN;
            ramp_adam_kernel<<<LRN_GRID, 256, 0, st>>>(aa, p->n_weights);
            CUDA_TRY(cudaGetLastError());
            launches += 6;
        }
    }
    if (cfg->num_sgd_iter > 0) p->emb_valid = false;
    p->b_rows = rows;
    // 5. the last pass's statistics and the adapted KL coefficient: the call's one read-back
    ramp_ppo_learn_stats_kernel<<<1, 1, 0, st>>>(p->l_mb_stats.get(), cfg->num_sgd_iter > 0 ? n_mb : 0, (float)cfg->kl_coeff,
                                                 (float)cfg->kl_target, p->l_n_rows.get(), p->l_stats.get());
    CUDA_TRY(cudaGetLastError());
    ramp_internal_count_launches(eng, launches + 1);
    if (stats_out) CUDA_TRY(cudaMemcpyAsync(stats_out, p->l_stats.get(), sizeof(double) * RAMP_PPO_STATS_LEN, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

int ramp_policy_train_batch_read(ramp_policy_t* p, ramp_engine_t* eng, int32_t* n_out, int32_t* model_out, int32_t* action_out,
                                 float* logp_out, float* logp_old_out, float* advantage_out, float* value_target_out) {
    if (!p || !eng || !n_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (p->b_rows < 1) return set_error(RAMP_ERR_BAD_ARG, "ppo: no train batch (ramp_policy_learn / ramp_policy_learn_pg)");
    cudaStream_t st = ramp_internal_stream(eng);
    CUDA_TRY(cudaMemcpyAsync(n_out, p->l_n_rows.get(), sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    const size_t n = (size_t)*n_out;
    if (model_out) CUDA_TRY(cudaMemcpyAsync(model_out, p->b_model.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    if (action_out) CUDA_TRY(cudaMemcpyAsync(action_out, p->b_action.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    if (logp_out) CUDA_TRY(cudaMemcpyAsync(logp_out, p->b_logp.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    if (logp_old_out) CUDA_TRY(cudaMemcpyAsync(logp_old_out, p->b_logp_old.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    if (advantage_out) CUDA_TRY(cudaMemcpyAsync(advantage_out, p->b_adv.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    if (value_target_out) CUDA_TRY(cudaMemcpyAsync(value_target_out, p->b_vt.get(), 4 * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

int ramp_policy_learner_state(ramp_policy_t* p, float* exp_avg_out, float* exp_avg_sq_out, int32_t* step_out) {
    if (!p) return set_error(RAMP_ERR_BAD_ARG, "null policy");
    CUDA_TRY(cudaSetDevice(p->device));
    if (!p->learner_ready) {
        if (exp_avg_out) memset(exp_avg_out, 0, sizeof(float) * p->n_weights);
        if (exp_avg_sq_out) memset(exp_avg_sq_out, 0, sizeof(float) * p->n_weights);
        if (step_out) *step_out = 0;
        return RAMP_OK;
    }
    CUDA_TRY(cudaDeviceSynchronize());                                    // a learn call may still be updating them
    if (exp_avg_out) CUDA_TRY(cudaMemcpy(exp_avg_out, p->l_adam_m.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToHost));
    if (exp_avg_sq_out) CUDA_TRY(cudaMemcpy(exp_avg_sq_out, p->l_adam_v.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToHost));
    if (step_out) CUDA_TRY(cudaMemcpy(step_out, p->l_step.get() + p->adam_parity, sizeof(int32_t), cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_policy_learner_reset(ramp_policy_t* p) {
    if (!p) return set_error(RAMP_ERR_BAD_ARG, "null policy");
    CUDA_TRY(cudaSetDevice(p->device));
    if (!p->learner_ready) return RAMP_OK;
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemset(p->l_adam_m.get(), 0, sizeof(float) * p->n_weights));
    CUDA_TRY(cudaMemset(p->l_adam_v.get(), 0, sizeof(float) * p->n_weights));
    CUDA_TRY(cudaMemset(p->l_step.get(), 0, sizeof(int32_t) * 2));
    return RAMP_OK;
}

int ramp_impala_loss_grad(ramp_policy_t* p, const ramp_impala_config_t* cfg, int32_t n_fragments, int32_t fragment_length,
                          const int32_t* model, const float* graph_features, const uint8_t* action_mask, const int32_t* action,
                          const float* behaviour_logp, const double* reward, const uint8_t* done, float* grad_out,
                          double* stats_out, float* vs_out, float* pg_adv_out, float* log_rho_out) {
    if (!p || !model || !graph_features || !action_mask || !action || !behaviour_logp || !reward || !done)
        return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_impala_config(cfg);
    if (rc != RAMP_OK) return rc;
    if (n_fragments < 1 || fragment_length < 1 || (int64_t)n_fragments * fragment_length > INT32_MAX)
        return set_error(RAMP_ERR_BAD_ARG, "impala: loss of %d fragments of %d rows", n_fragments, fragment_length);
    const int32_t n = n_fragments * fragment_length;
    CUDA_TRY(cudaSetDevice(p->device));
    if ((rc = prepare_learner(p, 0)) || (rc = ensure_rows(p, n)) || (rc = ensure_impala(p, n, 1)) ||
        (rc = upload_host_batch(p, n, model, graph_features, action_mask, nullptr, nullptr, action, nullptr, nullptr, nullptr)))
        return rc;
    CUDA_TRY(cudaMemcpy(p->i_blogp.get(), behaviour_logp, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(p->i_reward.get(), reward, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(p->i_done.get(), done, (size_t)n, cudaMemcpyHostToDevice));
    if ((rc = launch_states(p, 0, nullptr, 0, nullptr)) != RAMP_OK) return rc;
    GradArgs ga = host_batch_args(p, n);
    if ((rc = impala_batch(p, 0, *cfg, fragment_length, 0, n_fragments, nullptr, p->h_gf.get(), p->h_model.get(), p->h_mask.get(),
                           p->h_action.get(), p->i_blogp.get(), p->i_reward.get(), p->i_done.get(), ga, p->i_stats.get())) != RAMP_OK)
        return rc;
    CUDA_TRY(cudaMemsetAsync(p->i_stats.get() + RAMP_IMPALA_SGD_STEPS, 0, sizeof(double), 0));
    CUDA_TRY(cudaStreamSynchronize(0));
    p->i_rows = n;
    if (grad_out) CUDA_TRY(cudaMemcpy(grad_out, p->l_grad.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToHost));
    if (stats_out) CUDA_TRY(cudaMemcpy(stats_out, p->i_stats.get(), sizeof(double) * RAMP_IMPALA_STATS_LEN, cudaMemcpyDeviceToHost));
    if (vs_out) CUDA_TRY(cudaMemcpy(vs_out, p->i_vs.get(), sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
    if (pg_adv_out) CUDA_TRY(cudaMemcpy(pg_adv_out, p->i_pg.get(), sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
    if (log_rho_out) CUDA_TRY(cudaMemcpy(log_rho_out, p->i_log_rho.get(), sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_policy_learn_impala(ramp_policy_t* p, ramp_engine_t* eng, int32_t n_steps, const ramp_impala_config_t* cfg, double* stats_out) {
    if (!p || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_impala_config(cfg);
    if (rc != RAMP_OK) return rc;
    ramp_env_buffers_t eb{};
    if ((rc = ramp_env_buffers(eng, &eb)) != RAMP_OK) return rc;
    if (n_steps < 1 || n_steps > p->traj_n)
        return set_error(RAMP_ERR_BAD_ARG, "impala: %d steps asked of a trajectory with %d recorded", n_steps, p->traj_n);
    if (eb.n_episodes != p->traj_b || eb.n_actions != p->traj_a)
        return set_error(RAMP_ERR_BAD_ARG, "impala: the trajectory was recorded from another environment");
    const int32_t L = cfg->rollout_fragment_length ? cfg->rollout_fragment_length : n_steps;
    if (n_steps % L) return set_error(RAMP_ERR_BAD_ARG, "impala: rollout_fragment_length %d does not divide %d steps", L, n_steps);
    if (cfg->train_batch_size < L)
        return set_error(RAMP_ERR_BAD_ARG, "impala: train_batch_size %d is below rollout_fragment_length %d", cfg->train_batch_size, L);
    const ramp_policy_config_t& c = p->P.c;
    CUDA_TRY(cudaSetDevice(p->device));
    cudaStream_t st = ramp_internal_stream(eng);
    const int32_t B = eb.n_episodes, n_frag = (n_steps / L) * B, R = n_steps * B;
    const int32_t F = std::min(cfg->train_batch_size / L, n_frag), mb = F * L, n_sgd = (n_frag + F - 1) / F;
    if ((rc = prepare_learner(p, st)) || (rc = ensure_rows(p, mb)) || (rc = ensure_impala(p, R, n_sgd))) return rc;
    // 1. the fragment rows, fragment-major
    ImpalaBatchArgs ba{};
    ba.T = n_steps; ba.B = B; ba.A = c.n_actions; ba.L = L; ba.n_models = c.n_models;
    ba.t_obs = p->t_obs.get(); ba.t_model = p->t_model.get(); ba.t_mask = p->t_mask.get(); ba.t_action = p->t_action.get();
    ba.t_logp = p->t_logp.get(); ba.t_reward = p->t_reward.get(); ba.t_done = p->t_done.get();
    ba.obs = p->i_obs.get(); ba.model = p->i_model.get(); ba.mask = p->i_mask.get(); ba.action = p->i_action.get();
    ba.blogp = p->i_blogp.get(); ba.reward = p->i_reward.get(); ba.done = p->i_done.get(); ba.n_rows = p->i_n_rows.get();
    ramp_impala_batch_kernel<<<(unsigned)((R + 255) / 256), 256, 0, st>>>(ba);
    CUDA_TRY(cudaGetLastError());
    // 2. one SGD step per train batch, in order
    AdamArgs aa{};
    aa.lr = cfg->lr; aa.beta1 = cfg->adam_beta1; aa.beta2 = cfg->adam_beta2;
    aa.beta2_f = (float)cfg->adam_beta2; aa.one_m_beta1 = (float)(1.0 - cfg->adam_beta1); aa.one_m_beta2 = (float)(1.0 - cfg->adam_beta2);
    aa.eps = (float)cfg->adam_eps;
    aa.max_norm = (float)cfg->grad_clip; aa.n_rows = p->i_n_rows.get(); aa.mb = mb; aa.step = p->l_step.get();
    aa.m = p->l_adam_m.get(); aa.v = p->l_adam_v.get(); aa.grad = p->l_grad.get(); aa.norm_part = p->l_norm_part.get(); aa.w = p->d_w.get();
    aa.row_stats = nullptr; aa.stats = p->i_stats.get();             // IMPALA's statistics: ramp_impala_step_stats_kernel
    for (int k = 0; k < n_sgd; ++k) {
        const int32_t start = k * mb, nf = std::min(F, n_frag - k * F);
        // the rounds at the current weights, kept for the backward; from the second step on also the embeddings, which the
        // previous update made stale (the first uses those the trajectory was collected with)
        if ((rc = launch_states(p, st, p->i_n_rows.get(), start, k ? p->d_emb.get() : nullptr)) != RAMP_OK) return rc;
        GradArgs ga{};
        ga.mb = mb; ga.start = start; ga.n_rows = p->i_n_rows.get();
        if ((rc = impala_batch(p, st, *cfg, L, start, nf, p->i_obs.get(), nullptr, p->i_model.get(), p->i_mask.get(), p->i_action.get(),
                               p->i_blogp.get(), p->i_reward.get(), p->i_done.get(), ga,
                               p->i_step_stats.get() + (size_t)k * RAMP_IMPALA_STATS_LEN)) != RAMP_OK)
            return rc;
        aa.start = start;
        aa.parity = p->adam_parity; p->adam_parity ^= 1;
        ramp_adam_kernel<<<LRN_GRID, 256, 0, st>>>(aa, p->n_weights);
        CUDA_TRY(cudaGetLastError());
    }
    p->emb_valid = false;
    p->i_rows = R;
    // 3. the means over the steps: the call's one read-back
    ramp_impala_learn_stats_kernel<<<1, 1, 0, st>>>(p->i_step_stats.get(), n_sgd, p->i_stats.get());
    CUDA_TRY(cudaGetLastError());
    ramp_internal_count_launches(eng, 2 + 9 * n_sgd);
    if (stats_out) CUDA_TRY(cudaMemcpyAsync(stats_out, p->i_stats.get(), sizeof(double) * RAMP_IMPALA_STATS_LEN, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

int ramp_impala_vtrace_read(ramp_policy_t* p, int32_t* n_out, float* target_logp_out, float* log_rho_out, float* vs_out,
                            float* pg_adv_out) {
    if (!p || !n_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (p->i_rows < 1) return set_error(RAMP_ERR_BAD_ARG, "impala: no V-trace yet (ramp_policy_learn_impala / ramp_impala_loss_grad)");
    CUDA_TRY(cudaSetDevice(p->device));
    CUDA_TRY(cudaDeviceSynchronize());
    const size_t n = (size_t)p->i_rows;
    *n_out = p->i_rows;
    if (target_logp_out) CUDA_TRY(cudaMemcpy(target_logp_out, p->i_tlogp.get(), 4 * n, cudaMemcpyDeviceToHost));
    if (log_rho_out) CUDA_TRY(cudaMemcpy(log_rho_out, p->i_log_rho.get(), 4 * n, cudaMemcpyDeviceToHost));
    if (vs_out) CUDA_TRY(cudaMemcpy(vs_out, p->i_vs.get(), 4 * n, cudaMemcpyDeviceToHost));
    if (pg_adv_out) CUDA_TRY(cudaMemcpy(pg_adv_out, p->i_pg.get(), 4 * n, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

// pg_torch_policy.py pg_torch_loss: -mean(logp(a) advantages) over the train batch, on host rows
int ramp_pg_loss_grad(ramp_policy_t* p, const ramp_pg_config_t* cfg, int32_t n, const int32_t* model, const float* graph_features,
                      const uint8_t* action_mask, const int32_t* action, const float* advantage, float* grad_out, double* stats_out) {
    if (!p || !model || !graph_features || !action_mask || !action || !advantage) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_pg_config(cfg);
    if (rc != RAMP_OK) return rc;
    if (n < 1) return set_error(RAMP_ERR_BAD_ARG, "pg: loss of %d rows", n);
    CUDA_TRY(cudaSetDevice(p->device));
    if ((rc = prepare_learner(p, 0)) || (rc = ensure_rows(p, n)) ||
        (rc = upload_host_batch(p, n, model, graph_features, action_mask, nullptr, nullptr, action, nullptr, advantage, nullptr)))
        return rc;
    GradArgs ga = host_batch_args(p, n);
    ga.pg = 1; ga.action = p->h_action.get(); ga.adv = p->h_adv.get();
    if ((rc = launch_states(p, 0, nullptr, 0, nullptr)) != RAMP_OK || (rc = launch_grad(p, ga, 0)) != RAMP_OK) return rc;
    ramp_pg_stats_kernel<<<1, 1>>>(p->l_row_stats.get(), p->l_row_model.get(), p->h_adv.get(), n, ga.n_rows, p->l_norm_part.get(), p->l_stats.get());
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(0));
    if (grad_out) CUDA_TRY(cudaMemcpy(grad_out, p->l_grad.get(), sizeof(float) * p->n_weights, cudaMemcpyDeviceToHost));
    if (stats_out) CUDA_TRY(cudaMemcpy(stats_out, p->l_stats.get(), sizeof(double) * RAMP_PG_STATS_LEN, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

// PG's training step (algorithms/pg: one learn_on_batch per train batch): post_process_advantages (compute_advantages with
// use_gae False, use_critic False, last_r 0), pg_torch_loss, torch.optim.Adam
int ramp_policy_learn_pg(ramp_policy_t* p, ramp_engine_t* eng, int32_t n_steps, const ramp_pg_config_t* cfg, double* stats_out) {
    if (!p || !eng) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    int rc = check_pg_config(cfg);
    if (rc != RAMP_OK) return rc;
    ramp_env_buffers_t eb{};
    if ((rc = ramp_env_buffers(eng, &eb)) != RAMP_OK) return rc;
    if (n_steps < 1 || n_steps > p->traj_n)
        return set_error(RAMP_ERR_BAD_ARG, "pg: %d steps asked of a trajectory with %d recorded", n_steps, p->traj_n);
    if (eb.n_episodes != p->traj_b || eb.n_actions != p->traj_a)
        return set_error(RAMP_ERR_BAD_ARG, "pg: the trajectory was recorded from another environment");
    const ramp_policy_config_t& c = p->P.c;
    CUDA_TRY(cudaSetDevice(p->device));
    cudaStream_t st = ramp_internal_stream(eng);
    const int32_t B = eb.n_episodes, rows = n_steps * B;
    if ((rc = prepare_learner(p, st)) || (rc = ensure_rows(p, rows)) || (rc = ensure_batch(p, rows))) return rc;
    // 1. the discounted returns (ramp_ppo_gae_kernel without values: lambda 1, V = 0, a 0 bootstrap), the live rows t-major
    GaeArgs ge{};
    ge.T = n_steps; ge.B = B; ge.A = c.n_actions; ge.n_models = c.n_models; ge.standardize = 0;
    ge.gamma = cfg->gamma; ge.lambda = 1.0;
    ge.t_obs = p->t_obs.get(); ge.t_model = p->t_model.get(); ge.t_mask = p->t_mask.get(); ge.t_action = p->t_action.get();
    ge.t_logp = p->t_logp.get(); ge.t_value = nullptr; ge.t_reward = p->t_reward.get(); ge.t_done = p->t_done.get();
    ge.boot = nullptr; ge.adv64 = p->b_adv64.get();
    ge.obs = p->b_obs.get(); ge.model = p->b_model.get(); ge.mask = p->b_mask.get(); ge.action = p->b_action.get(); ge.logp = p->b_logp.get();
    ge.adv = p->b_adv.get(); ge.vt = p->b_vt.get(); ge.n_rows = p->l_n_rows.get();
    ramp_ppo_gae_kernel<<<1, 1024, 0, st>>>(ge);
    CUDA_TRY(cudaGetLastError());
    // 2. the loss's gradient over the whole batch at the collection weights (the embeddings the trajectory was collected with);
    //    the log p(a) the gradient kernel recomputes goes to b_logp_old
    GradArgs ga{};
    ga.mb = rows; ga.start = 0; ga.n_rows = p->l_n_rows.get(); ga.shuffle = 0; ga.obs_dyn = p->b_obs.get(); ga.model = p->b_model.get();
    ga.mask = p->b_mask.get(); ga.action = p->b_action.get(); ga.adv = p->b_adv.get(); ga.pg = 1; ga.logp_old = p->b_logp_old.get();
    if ((rc = launch_states(p, st, p->l_n_rows.get(), 0, nullptr)) != RAMP_OK || (rc = launch_grad(p, ga, st)) != RAMP_OK) return rc;
    // 3. one Adam step; with no row in the batch, none (the step count stays)
    AdamArgs aa{};
    aa.lr = cfg->lr; aa.beta1 = cfg->adam_beta1; aa.beta2 = cfg->adam_beta2;
    aa.beta2_f = (float)cfg->adam_beta2; aa.one_m_beta1 = (float)(1.0 - cfg->adam_beta1); aa.one_m_beta2 = (float)(1.0 - cfg->adam_beta2);
    aa.eps = (float)cfg->adam_eps;
    aa.max_norm = (float)cfg->grad_clip; aa.n_rows = p->l_n_rows.get(); aa.mb = rows; aa.start = 0; aa.step = p->l_step.get();
    aa.m = p->l_adam_m.get(); aa.v = p->l_adam_v.get(); aa.grad = p->l_grad.get(); aa.norm_part = p->l_norm_part.get(); aa.w = p->d_w.get();
    aa.row_stats = nullptr; aa.stats = p->l_stats.get();            // PG's statistics: ramp_pg_stats_kernel, after it
    aa.parity = p->adam_parity; p->adam_parity ^= 1;
    ramp_adam_kernel<<<LRN_GRID, 256, 0, st>>>(aa, p->n_weights);
    // 4. the statistics: the call's one read-back
    ramp_pg_stats_kernel<<<1, 1, 0, st>>>(p->l_row_stats.get(), p->l_row_model.get(), p->b_adv.get(), rows, p->l_n_rows.get(),
                                          p->l_norm_part.get(), p->l_stats.get());
    CUDA_TRY(cudaGetLastError());
    p->emb_valid = false;
    p->b_rows = rows;
    ramp_internal_count_launches(eng, 8);
    if (stats_out) CUDA_TRY(cudaMemcpyAsync(stats_out, p->l_stats.get(), sizeof(double) * RAMP_PG_STATS_LEN, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return RAMP_OK;
}

}  // extern "C"

#include "ramp_es.cuh"
