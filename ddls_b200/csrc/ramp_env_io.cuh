// ramp_env_io.cuh -- the device environment's i/o in caller-owned device memory (include/ramp_b200.h: ramp_env_ingest /
// ramp_env_export): actions in from a framework tensor, the reference's observation row, reward and done out.  Both kernels run on
// the caller's stream; ramp_engine.cu fences the engine stream around them.
//
//   ramp_env_ingest_kernel  one thread per episode: an int32 or int64 action -> the environment's int32 `actions`.  A value outside
//                           the action set [0, max_degree] never reaches ramp_env_decide_kernel: it is written as 0 and the first
//                           such live episode is recorded (RJPE:314-316 raises "Action a not in action set", whatever
//                           apply_action_mask says).  The call number that keys the record is on the device and advanced by the
//                           kernel, so a CUDA graph's replays number their calls as eager calls do
//   ramp_env_export_kernel  one thread per (episode, graph_features column): RampJobPartitioningObservation's graph_features row
//                           (ramp_job_partitioning_observation.py:275: the nine job features, the queued model's six per-graph
//                           statistics, mounted workers and running jobs, then the action mask as 0.0 / 1.0), plus model, mask,
//                           reward and done
#pragma once

namespace ramp {

constexpr int ENV_GF_JOB = 9;          // obs_dyn[0:9]: the queued job's normalised features (observation.py:358-498)
constexpr int ENV_GF_STATIC = 6;       // mean / median of op compute, op memory and dep size (observation.py:425-469)
constexpr int ENV_GF_BASE = 17;        // graph_features columns before the action mask
constexpr unsigned long long ENV_NO_RANGE_ERR = ~0ull;

struct EnvIngestArgs {
    const void* actions;               // caller's [B] int32 (is64 = 0) or int64 (is64 = 1)
    int32_t is64, B, max_degree;
    uint32_t* seq;                     // [2]: the ingest call number since the error word was last cleared, and the CTAs of this
                                       // call that are done with it; the call's last CTA advances the number (a replayed CUDA
                                       // graph runs no host code, so the number lives here)
    const uint8_t* done;               // [B] EnvDev::done
    int32_t* out;                      // [B] EnvDev::actions
    unsigned long long* range_err;     // (seq << 32) | episode of the first out-of-set action, ENV_NO_RANGE_ERR when none
    long long* range_val;              // [B] the action recorded with it
};

__global__ void ramp_env_ingest_kernel(const EnvIngestArgs a) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < a.B) {
        const long long x = a.is64 ? static_cast<const long long*>(a.actions)[b] : (long long)static_cast<const int32_t*>(a.actions)[b];
        const bool in_set = x >= 0 && x <= a.max_degree;
        a.out[b] = in_set ? (int32_t)x : 0;
        if (!in_set && !a.done[b]) {                                                 // RJPE:314-316 looks at the live episodes
            // the word is sticky: an error of an earlier call (stream order makes its key visible here) stays the one reported.
            // Within one call the lowest episode wins, and only thread b writes range_val[b]
            const uint32_t seq = a.seq[0];
            const unsigned long long cur = *(volatile unsigned long long*)a.range_err;
            if (cur == ENV_NO_RANGE_ERR || (uint32_t)(cur >> 32) == seq) {
                a.range_val[b] = x;
                atomicMin(a.range_err, ((unsigned long long)seq << 32) | (unsigned)b);
            }
        }
    }
    // every thread of the CTA has read the number; the last CTA to get here advances it for the next call
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(a.seq + 1, 1u) == gridDim.x - 1) {
            a.seq[1] = 0;
            a.seq[0] += 1;
        }
    }
}

struct EnvExportArgs {
    int32_t B, A, n_models;
    const int32_t* queued_model; const float* obs_dyn; const uint8_t* mask; const double* reward; const uint8_t* done;   // EnvDev
    const float* graph_static;         // [n_models][6]
    long long* model;                  // [B] or null
    float* graph_features;             // [B][17 + A] or null
    uint8_t* action_mask;              // [B][A] or null (0 / 1: torch.bool)
    double* reward_out;                // [B] or null
    uint8_t* done_out;                 // [B] or null (0 / 1)
};

__global__ void ramp_env_export_kernel(const EnvExportArgs a) {
    const int C = ENV_GF_BASE + a.A;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)a.B * C) return;
    const int b = (int)(i / C), c = (int)(i - (long long)b * C);
    const int k = c - ENV_GF_BASE;                                                   // action of a mask column
    if (a.graph_features) {
        float x;
        if (c < ENV_GF_JOB) {
            x = a.obs_dyn[(size_t)b * 11 + c];
        } else if (c < ENV_GF_JOB + ENV_GF_STATIC) {
            const int m = a.queued_model[b];
            x = (m >= 0 && m < a.n_models) ? a.graph_static[m * ENV_GF_STATIC + (c - ENV_GF_JOB)] : 0.f;
        } else if (c < ENV_GF_BASE) {
            x = a.obs_dyn[(size_t)b * 11 + (c - ENV_GF_STATIC)];                    // columns 15, 16: obs_dyn[9], obs_dyn[10]
        } else {
            x = a.mask[(size_t)b * a.A + k] ? 1.f : 0.f;
        }
        a.graph_features[i] = x;
    }
    if (k >= 0 && a.action_mask) a.action_mask[(size_t)b * a.A + k] = a.mask[(size_t)b * a.A + k] ? 1 : 0;
    if (c == 0) {
        if (a.model) a.model[b] = a.queued_model[b];
        if (a.reward_out) a.reward_out[b] = a.reward[b];
        if (a.done_out) a.done_out[b] = a.done[b] ? 1 : 0;
    }
}

}  // namespace ramp
