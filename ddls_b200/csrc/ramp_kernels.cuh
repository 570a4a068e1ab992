// ramp_kernels.cuh -- device-side data layout and kernels of the GPU-native (H100, sm_90a) RAMP simulator hot path.
//
// Reference semantics (cwfparsonson/ddls @ 9e0b5ba; RCE = ddls/environments/ramp_cluster/
// ramp_cluster_environment.py, JOB = ddls/demands/jobs/job.py):
//   ramp_plan_kernel       memo lookup/insert of _perform_lookahead_job_completion_time   RCE:469-518, 269-275
//   ramp_lookahead_kernel  _run_lookahead tick loop                                        RCE:379-467
//   ramp_step_kernel       step(): block/mount/register lookahead/outer event loop/stats    RCE:894-1167
//
// All simulation arithmetic is IEEE f64 without FMA contraction (compile with -fmad=false), in the
// reference's accumulation order, so results are bit-identical to CPython floats.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <type_traits>

#include "../../include/ramp_b200.h"

namespace ramp {

// ---------------------------------------------------------------------------------------------------
// HBM layout

// One registered lowered job, in the layout the tick loop streams.  All arrays live in one device allocation
// (256 B aligned segments) and are read-only for the kernels.
//
// Priorities are pre-ranked on the host into unique u32 keys (larger wins): sorting by (priority desc, index asc)
// reproduces "iterate in sorted() order, replace only on strictly greater priority" (RCE:56-66, RCE:672-685), so
// the per-worker / per-channel arg-max is one 32-bit shared-memory atomicMax per item.  Everything a ready
// item needs is packed into a self-contained record, so the tick loop never gathers through an index:
//   op record  = { f64 remaining, u32 key, u32 worker } + { i32 first out-edge, i32 out-degree }   (24 B)
//   dep record = { u64 key | channel | is_flow | n_parents(child) | child op } + { f64 remaining }  (16 B)
struct TemplateDev {
    int32_t n_ops, n_deps, n_workers, n_channels;
    int32_t num_training_steps, model_id, degree, n_src;
    int32_t canon_id;           // id of the first registered byte-identical template (exact memo key)
    int32_t size_class;         // 0: small (one warp per lookahead is fastest), 1: big (one CTA per lookahead is fastest),
                                // 2: resident (quotient blob in shared memory, one THREAD per lookahead)
    int32_t par_in_smem;        // parent counters fit the shared-memory byte counters (max in-degree <= 255, N <= par_cap)
    int32_t _pad0;
    const int4*     op_rec;       // [N] by op index: {cost.lo, cost.hi, key, worker}
    const int2*     op_row;       // [N] by op index: {first out-edge, out-degree} (CSR row)
    const uint16_t* op_n_parents; // [N] by op index (JOB:508-523)
    const double*   dep_rt;       // [E] by dep index: init_run_time (RCE:542-560)
    const unsigned long long* dep_kd;  // [E] by dep index (CSR order): the whole dep in one word:
                                       //     key | channel << kd_cshift | is_flow << kd_fshift | n_parents(child) << (kd_fshift+1)
                                       //     | child op << kd_dshift; channel == kd_cmask means "none" (non-flows); the n_parents byte
                                       //     only when par_in_smem, i.e. every in-degree <= 255
    uint32_t kd_kmask, kd_cmask;  // (1 << key bits) - 1, (1 << channel bits) - 1
    int32_t  kd_cshift, kd_fshift, kd_dshift, _pad1;
    const int32_t*  src_ops;      // [n_src] ops with in-degree 0: the initial ops_ready (JOB:474-481)
    uint64_t scratch_bytes;       // HBM-side dynamic state one running lookahead of this template may need
    uint64_t algorithmic_bytes_static; // 20 N + 19 E + 24 (SURVEY.md 8d), + 12 T added per run
    // symmetry quotient (ramp_quotient.cpp) packed for the thread-per-lookahead kernel (ramp_lookahead_thread.cuh): one blob
    // that is bulk-copied into shared memory; null when the job is not resident-eligible (size_class 0 / 1 then)
    const unsigned char* res_blob;
    int32_t res_bytes;            // multiple of 16
    int32_t res_n_ops, res_n_deps, _pad2;
};

struct WorkItem {
    int32_t template_id;
    int32_t slot;               // result slot
    int32_t episode;            // -1 for standalone runs
    int32_t n_mounted_workers;  // len(job.details['mounted_workers']) of the mounting job (RCE:832); 0 = the template's
};

// lookahead result slots (SoA); slot == memo hash-table position (+ B extra slots for RAMP_MEMO_OFF)
struct ResultSlots {
    double*   jct;
    double*   comm;
    double*   comp;
    int32_t*  n_ticks;
    int32_t*  status;
    int64_t*  trace_off;        // offset into the trace pool, -1 if none
    double*   util;             // mean_mounted_worker_utilisation_frac (RCE:830-832) for util_nmw mounted workers
    int32_t*  util_nmw;
};

struct TracePool {
    int32_t* n_active;          // [pool_len]
    double*  tick;              // [pool_len]
    unsigned long long* top;    // bump allocator (entries)
    uint64_t len;
};

struct Counters {               // the first four words are zeroed at the start of every step
    int32_t n_work;             // work list 0: small lookaheads (or all of them for standalone runs)
    int32_t work_cursor;
    int32_t n_work_big;         // work list 1: big lookaheads
    int32_t work_cursor_big;
    int32_t err_episode;        // first episode that recorded an error (+1), 0 if none
    int32_t err_status;
    int32_t n_work_res;         // work list 2: lookaheads on resident (quotient) templates; zeroed at the start of every step
    int32_t n_chunks;           // chunks ramp_bucket_kernel made of list 2
    int32_t chunk_cursor;
    int32_t _pad;
};

// ran: plan decisions that ran a lookahead (EI_PLAN_RAN = 1).  lookaheads counts every lookahead executed, including the
// speculative ones of overlapped steps whose episode turned out not to be live: lookaheads - ran of them went unused
struct MemoStats { unsigned long long lookups, hits, lookaheads, alg_bytes, shared_hits, quotient_bytes, ran; };

// running-job table fields (SoA: [field][row][episode])
// RF_COMM_FRAC / RF_COMP_FRAC: the job's comm / jct and comp / jct (RCE:962-982), divided once when it is mounted rather than
// in every tick of the outer event loop -- the same division of the same operands
enum { RF_JCT = 0, RF_STARTED, RF_COMM_FRAC, RF_COMP_FRAC, RF_UTIL, RF_PART_OP_MEM, RF_PART_DEP, RF_FLOW, RF_ORIG_OP_MEM,
       RF_ORIG_DEP, RF_COUNT };
enum { RI_JOB_IDX = 0, RI_N_WORKERS, RI_N_CHANNELS, RI_COUNT };

// per-episode scalars (SoA: [field][episode])
// EF_ACC_*: the episode_stats accumulators (RCE:1086-1106), every cluster step's values summed in cluster-step order --
// the seven *_info_processed in RAMP_SS_COMPUTE_INFO_PROCESSED order, the four step means RCE:1099-1102, the sums and length
// of the per-tick utilisation lists (RCE:1103-1104) and the number of cluster steps; ramp_episode_stats_kernel finalises them
enum { EF_NOW = 0, EF_NEXT_ARRIVAL, EF_LAST_ARRIVAL, EF_LOAD_SUM,
       EF_ACC_INFO, EF_ACC_COMP_FRAC = EF_ACC_INFO + 7, EF_ACC_COMM_FRAC, EF_ACC_JOBS_RUNNING, EF_ACC_MOUNTED_WORKERS,
       EF_ACC_UTIL_MOUNTED, EF_ACC_UTIL_CLUSTER, EF_ACC_TICKS, EF_ACC_STEPS, EF_COUNT };
// the env-step accumulators of EvalLoop's results['step_stats'] (eval_loop.py:50-100), next to the episode ones: RAMP_ESS_* and the
// env-step's tick count, opened by the action step, folded over every cluster step of the env-step in cluster-step order and closed
// into the env-step's row when it ends.  [B][ES_STRIDE]: one base address per episode, so that the fold adds no live registers to
// the step kernel (with the [field][B] layout of ef, ptxas keeps one address per field and spills)
enum { ES_TICKS = RAMP_ENV_STEP_STATS_LEN, ES_STRIDE };
enum { EI_NUM_ARRIVED = 0, EI_NUM_COMPLETED, EI_NUM_BLOCKED, EI_QUEUED, EI_N_RUNNING, EI_STEP_COUNTER, EI_EVENT_SEQ,
       EI_LOAD_N, EI_STATUS, EI_DONE, EI_LAST_SLOT, EI_PLAN_SLOT, EI_PLAN_RAN, EI_COUNT };

struct EpisodeState {
    int32_t B, max_running, max_jobs, n_jobs;
    int32_t n_cluster_workers, queue_capacity;
    double eps, max_sim_time;
    double*  ef;                // [EF_COUNT][B]
    double*  es;                // [B][ES_STRIDE] env-step accumulators; between env-steps the last env-step's row.  Null until
                                //     ramp_enable_env_step_stats: the step kernel then skips them
    int32_t* ei;                // [EI_COUNT][B]
    double*  rf;                // [RF_COUNT][max_running][B]
    int32_t* ri;                // [RI_COUNT][max_running][B]
    ramp_job_record_t* rec;     // [B][max_jobs]
    const ramp_arrival_t* arr;  // [B][max_jobs]
    double* tick_util;          // [B][tick_util_cap][2] or null: the step's per-tick utilisation lists (RCE:989-994), ramp_enable_tick_lists
    int32_t* tick_util_n;       // [B] their length in the last cluster step
    int32_t tick_util_cap;
    const int32_t* n_jobs_ep;   // [B] jobs the episode's arrival stream holds so far (len(jobs_generator) > 0 <=> more than arrived,
                                //     RCE:1019-1040); ramp_reset sets n_jobs for all, ramp_set_job_count changes one episode
};

struct MemoTable {
    unsigned long long* keys;   // [cap] 0 = empty
    uint32_t mask;              // cap - 1
    int32_t mode;
    // RAMP_MEMO_SHARED: level 1 = keys[] above (per episode) with vals[] -> result slot; level 2 = batch-wide cache
    int32_t* vals;              // [cap]
    unsigned long long* keys2;  // [cap2] keyed by the canonical (byte-identical) template id
    uint32_t mask2;
    int32_t slot2_base;         // result slot of level-2 position 0
};

struct LookaheadArgs {
    const TemplateDev* templates;
    const WorkItem* items;      // work list A, consumed first (the big lookaheads: longest-processing-time-first)
    const int32_t* n_work;      // device-side count of list A
    const WorkItem* items_b;    // work list B, consumed after A (may be null)
    const int32_t* n_work_b;    // device-side count of list B (may be null)
    int32_t* cursor;            // device-side work cursor over A then B (persistent warps / CTAs pull items)
    unsigned char* scratch;     // [gridDim.x][scratch_stride]
    uint64_t scratch_stride;
    ResultSlots res;
    TracePool pool;
    int32_t trace_cap;          // per-CTA temp trace capacity
    int32_t w_cap, c_cap;       // shared-memory key array capacities
    int32_t par_cap;            // bytes of shared-memory parent counters per lookahead (0 = none)
    MemoStats* stats;
};

__host__ __device__ inline uint64_t align_up(uint64_t x, uint64_t a) { return (x + a - 1) / a * a; }

// HBM-side dynamic state of one running lookahead, carved out of the owning warp's scratch slab.  The hot state
// (op frontier, the first RAMP_F_CAP entries of the dep frontier, per-worker / per-channel winners) lives in
// shared memory; HBM holds the parent counters, the overflow of the two frontiers and the tick trace.
struct ScratchView {
    uint32_t* par_done;              // [N] len(parent_deps_completed) JOB:530
    int4*     ops_a_ovf[2];          // [N] overflow of the shared-memory op frontier (ping-pong)
    int2*     ops_b_ovf[2];          // [N]
    unsigned long long* f_km_ovf;    // [E] overflow of the shared-memory dep frontier: packed dep words
    double*   f_rem_ovf;             // [E]                                              remaining times
    unsigned long long* f_km_ovf2;   // [E] second buffer (CTA-per-lookahead kernel compacts by ping-pong)
    double*   f_rem_ovf2;            // [E]
    unsigned long long* nf_ovf;      // [E] overflow of the shared-memory list of ready non-flow deps
    int32_t*  rq_ovf;                // [N] overflow of the CTA kernel's queue of ops readied in the current tick
    int32_t*  tr_n;                  // [trace_cap] temp trace
    double*   tr_tick;               // [trace_cap]
};

__host__ __device__ inline uint64_t scratch_bytes_for(int32_t N, int32_t E) {
    uint64_t b = 0;
    b += align_up((uint64_t)N * 4, 16);
    b += 2 * align_up((uint64_t)N * 16, 16);
    b += 2 * align_up((uint64_t)N * 8, 16);
    b += 5 * align_up((uint64_t)E * 8, 16);
    b += align_up((uint64_t)N * 4, 16);
    return b;
}

__device__ inline ScratchView carve(unsigned char* base, int32_t N, int32_t E, uint64_t trace_region_off, int32_t trace_cap) {
    ScratchView v;
    uint64_t o = 0;
    v.par_done = (uint32_t*)(base + o);              o += align_up((uint64_t)N * 4, 16);
    v.ops_a_ovf[0] = (int4*)(base + o);              o += align_up((uint64_t)N * 16, 16);
    v.ops_a_ovf[1] = (int4*)(base + o);              o += align_up((uint64_t)N * 16, 16);
    v.ops_b_ovf[0] = (int2*)(base + o);              o += align_up((uint64_t)N * 8, 16);
    v.ops_b_ovf[1] = (int2*)(base + o);              o += align_up((uint64_t)N * 8, 16);
    v.f_km_ovf = (unsigned long long*)(base + o);    o += align_up((uint64_t)E * 8, 16);
    v.f_rem_ovf = (double*)(base + o);               o += align_up((uint64_t)E * 8, 16);
    v.f_km_ovf2 = (unsigned long long*)(base + o);   o += align_up((uint64_t)E * 8, 16);
    v.f_rem_ovf2 = (double*)(base + o);              o += align_up((uint64_t)E * 8, 16);
    v.nf_ovf = (unsigned long long*)(base + o);      o += align_up((uint64_t)E * 8, 16);
    v.rq_ovf = (int32_t*)(base + o);                 o += align_up((uint64_t)N * 4, 16);
    v.tr_tick = (double*)(base + trace_region_off);
    v.tr_n = (int32_t*)(v.tr_tick + trace_cap);
    return v;
}

// ---------------------------------------------------------------------------------------------------
// small device helpers

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

// Python: x -= min(tick, x) (JOB:555, JOB:561); min(a, b) returns a unless b < a.
__device__ __forceinline__ double tick_down(double rem, double tick) {
    const double m = (rem < tick) ? rem : tick;
    return __dsub_rn(rem, m);
}

// min over the warp of NON-NEGATIVE doubles (remaining times; +inf = "none"): their u64 bit patterns order like the
// values, so two 32-bit REDUX.MIN (high word, then low word among the lanes holding the minimal high word) replace a
// ten-shuffle butterfly
__device__ __forceinline__ double warp_min_f64(double v) {
    const unsigned hi = (unsigned)__double2hiint(v), lo = (unsigned)__double2loint(v);
    const unsigned mh = __reduce_min_sync(0xffffffffu, hi);
    const unsigned ml = __reduce_min_sync(0xffffffffu, hi == mh ? lo : 0xffffffffu);
    return __hiloint2double((int)mh, (int)ml);
}

__device__ __forceinline__ int warp_sum_i32(int v) {
    return __reduce_add_sync(0xffffffffu, v);
}

#define RAMP_INF_BITS 0x7FF0000000000000ull

// RCE:830-832: util = sum over ticks, in tick order, of (n_active / n_mounted_workers) * (tick / jct).  The divisions
// and the product of every term are independent, so `n_threads` threads compute them (into term[]), then ONE thread
// adds them serially in tick order -- the same f64 additions in the same order as the reference.
__device__ __forceinline__ void util_terms(const int32_t* tr_n, const double* tr_tick, double* term, int n_rec, double nmw,
                                            double jct, int tid, int n_threads) {
    for (int k = tid; k < n_rec; k += n_threads)
        term[k] = __dmul_rn(__ddiv_rn((double)tr_n[k], nmw), __ddiv_rn(tr_tick[k], jct));
}
__device__ __forceinline__ double util_sum(const double* term, int n_rec) {
    double u = 0.0;
    for (int k = 0; k < n_rec; ++k) u = __dadd_rn(u, term[k]);
    return u;
}

// ---------------------------------------------------------------------------------------------------
// _run_lookahead (RCE:379-467): ONE WARP per lookahead; WPB independent warps per CTA; persistent warps pull
// work items from a device-side cursor.  No block barriers: per-tick frontiers are tens to hundreds of
// items, so a warp keeps its lanes busy and all cross-lane traffic is shuffles / ballots / shared atomics.
// A lone warp is bound by dependent memory round trips, so the ready frontiers are staged in shared memory
// (HBM only on overflow) and the remaining global phases issue a whole batch of loads before consuming any.
//
// Per tick (letters as in SURVEY.md 3.3):
//   A  per-worker arg-max over ready ops           -> atomicMax of rank keys into smem wkey[]      (RCE:562-590, 44-67)
//   B  t_op = min remaining over the op winners    -> REDUX.MIN on the f64 bit pattern              (RCE:592-606)
//   C  any ready non-flow dep?  They sit in their own list: run time zero (RCE:542-560), so each lives for exactly one
//      tick, and a tick that finds the list non-empty is the reference's zero-length tick (RCE:412-422, 718-731): it
//      completes exactly those and leaves the flows and the channel winners untouched                  (RCE:520-540)
//   D  t_comm = min remaining over the per-channel winners.  The per-channel arg-max (RCE:608-629, 665-689) is kept in a
//      DOUBLE-BUFFERED table: while a tick runs, every flow that survives it and every flow that arrives votes (atomicMax
//      of its key) into the next tick's table, so the table is always complete and never needs a rescan when a winner
//      completes.  D is one pass over the ready flows: the winners are the entries whose key equals ck_cur[channel]. (RCE:653-663)
//   E  tick = min(t_op, t_comm)                                                                     (RCE:426)
//   H  every flow of the pre-tick snapshot: rem -= min(tick, rem); == 0 -> completed: atomicAdd on the child's parent
//      counter, == n_parents -> the child is readied (its op index is queued; the 24-byte records of all ops readied in
//      the tick are fetched in ONE batch, the loads overlapping G).  Survivors are slid down in place. (RCE:733-775)
//   G  op winners: same; completed -> the CSR rows of all ops completed in this tick are appended to the flow frontier /
//      the non-flow list as one flattened, coalesced copy (first ticked next tick == the RCE:429 snapshot). (RCE:691-716)
//   I,J lane 0 accumulates t / comm / comp and the trace in tick order                              (RCE:442-445, 777-791)
#ifndef RAMP_U
#define RAMP_U 2            // batch depth: independent loads in flight per lane per phase
#endif
#ifndef RAMP_OPS_CAP
#define RAMP_OPS_CAP 48     // op-frontier records kept in shared memory per buffer (overflow goes to HBM)
#endif
#ifndef RAMP_F_CAP
#define RAMP_F_CAP 384      // flow-frontier entries kept in shared memory (overflow goes to HBM); sized so that 12 lookahead warps fit an SM
#endif

#ifndef RAMP_NF_CAP
#define RAMP_NF_CAP 64      // ready non-flow deps kept in shared memory (they live for exactly one tick)
#endif

struct OpsView { int4* a_sm; int2* b_sm; int4* a_ovf; int2* b_ovf; };
template <int OC = RAMP_OPS_CAP>
__device__ __forceinline__ void ops_get(const OpsView& v, int k, int4& ra, int2& rb) {
    if (k < OC) { ra = v.a_sm[k]; rb = v.b_sm[k]; } else { ra = v.a_ovf[k - OC]; rb = v.b_ovf[k - OC]; }
}
template <int OC = RAMP_OPS_CAP>
__device__ __forceinline__ void ops_put(const OpsView& v, int k, const int4 ra, const int2 rb) {
    if (k < OC) { v.a_sm[k] = ra; v.b_sm[k] = rb; } else { v.a_ovf[k - OC] = ra; v.b_ovf[k - OC] = rb; }
}
// dep frontier entry = the packed dep word (TemplateDev::dep_kd) + the remaining time: 16 B
// a readied op is first recorded as its op index only (in the row slot); its 24-byte record is fetched later, all
// records of a tick in one batch, so that the tick waits for ONE L2 round trip instead of one per 32-dep group
template <int OC = RAMP_OPS_CAP>
__device__ __forceinline__ void ops_put_child(const OpsView& v, int k, int child) {
    if (k < OC) v.b_sm[k] = make_int2(child, 0); else v.b_ovf[k - OC] = make_int2(child, 0);
}
template <int OC = RAMP_OPS_CAP>
__device__ __forceinline__ int ops_get_child(const OpsView& v, int k) {
    return (k < OC) ? v.b_sm[k].x : v.b_ovf[k - OC].x;
}

struct FrontView { unsigned long long* kd_sm; double* rem_sm; unsigned long long* kd_ovf; double* rem_ovf; };
template <int FC = RAMP_F_CAP>
__device__ __forceinline__ void f_get(const FrontView& v, int k, unsigned long long& kd, double& rem) {
    if (k < FC) { kd = v.kd_sm[k]; rem = v.rem_sm[k]; } else { kd = v.kd_ovf[k - FC]; rem = v.rem_ovf[k - FC]; }
}
template <int FC = RAMP_F_CAP>
__device__ __forceinline__ void f_put(const FrontView& v, int k, unsigned long long kd, double rem) {
    if (k < FC) { v.kd_sm[k] = kd; v.rem_sm[k] = rem; } else { v.kd_ovf[k - FC] = kd; v.rem_ovf[k - FC] = rem; }
}

// parent counter of op `child` += 1, returns the new value (JOB:530).  Small jobs keep one BYTE per op in shared memory
// (four per word, atomicAdd of 1 << 8*(child&3): a byte never carries because it never exceeds the in-degree <= 255)
__device__ __forceinline__ uint32_t par_inc(bool in_smem, uint32_t* par_sm, uint32_t* par_gl, int child) {
    if (in_smem) {
        const uint32_t sh = ((uint32_t)child & 3u) * 8u;
        const uint32_t old = atomicAdd(&par_sm[child >> 2], 1u << sh);
        return ((old >> sh) & 0xFFu) + 1u;
    }
    return atomicAdd(&par_gl[child], 1u) + 1u;
}

// bytes of shared memory one lookahead warp needs
__host__ __device__ inline size_t lookahead_smem_per_warp(int w_cap, int c_cap, int par_cap, int f_cap = RAMP_F_CAP, int ops_cap = RAMP_OPS_CAP) {
    size_t b = 0;
    b += (size_t)2 * ops_cap * 16;               // op records a (ping-pong)
    b += (size_t)f_cap * 8 * 2;                  // kd, rem
    b += (size_t)RAMP_NF_CAP * 8;                // ready non-flow deps
    b += (size_t)2 * ops_cap * 8;                // op records b
    b += (size_t)(w_cap + 2 * c_cap) * 4;        // wkey, ckey (this tick / next tick)
    b += (size_t)par_cap;                        // parent counters (bytes)
    return (b + 15) & ~(size_t)15;
}

// FC / OC: flow-frontier entries / op-frontier records kept in shared memory per warp.  The engine instantiates a roomy
// shape (384 / 48: 12 warps per SM) and a dense one (256 / 32: 16 warps per SM) for steps with far more lookaheads than slots
template <int WPB, int FC = RAMP_F_CAP, int OC = RAMP_OPS_CAP>
__global__ void __launch_bounds__(WPB * 32) ramp_lookahead_kernel(const LookaheadArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const unsigned lt_mask = (1u << lane) - 1u;
    unsigned char* my_smem = smem_raw + (size_t)warp * lookahead_smem_per_warp(a.w_cap, a.c_cap, a.par_cap, FC, OC);
    // layout by decreasing alignment: int4 | 8-byte arrays | 4-byte arrays
    int4* ops_a_sm0 = reinterpret_cast<int4*>(my_smem);                                  // [2][OC]
    FrontView fr;
    fr.kd_sm = reinterpret_cast<unsigned long long*>(ops_a_sm0 + 2 * OC);      // [FC]
    fr.rem_sm = reinterpret_cast<double*>(fr.kd_sm + FC);                        // [FC]
    unsigned long long* nf_sm = reinterpret_cast<unsigned long long*>(fr.rem_sm + FC);   // [RAMP_NF_CAP]
    int2* ops_b_sm0 = reinterpret_cast<int2*>(nf_sm + RAMP_NF_CAP);                      // [2][OC]
    uint32_t* wkey = reinterpret_cast<uint32_t*>(ops_b_sm0 + 2 * OC);          // [w_cap] best key among the ready ops on the worker
    uint32_t* ckey0 = wkey + a.w_cap;                                                    // [2][c_cap] best key among the ready flows on the channel
    uint32_t* par_sm = ckey0 + 2 * a.c_cap;                                              // [par_cap / 4] byte parent counters

    unsigned char* slab = a.scratch + (uint64_t)(blockIdx.x * WPB + warp) * a.scratch_stride;
    const uint64_t trace_region = a.scratch_stride - align_up((uint64_t)a.trace_cap * 12, 16);
    const double INF = __longlong_as_double(RAMP_INF_BITS);

    for (;;) {
        int wi = 0;
        if (lane == 0) wi = atomicAdd(a.cursor, 1);
        wi = __shfl_sync(FULL, wi, 0);
        const int n_a = *a.n_work;
        const int n_b = a.n_work_b ? *a.n_work_b : 0;
        if (wi >= n_a + n_b) break;
        const WorkItem item = (wi < n_a) ? a.items[wi] : a.items_b[wi - n_a];
        const TemplateDev& T = a.templates[item.template_id];
        const int N = T.n_ops, E = T.n_deps, W = T.n_workers, C = T.n_channels;
        const ScratchView sv = carve(slab, N, E, trace_region, a.trace_cap);
        fr.kd_ovf = sv.f_km_ovf; fr.rem_ovf = sv.f_rem_ovf;
        unsigned long long* nf_ovf = sv.nf_ovf;

        const int4* __restrict__ t_op_rec = T.op_rec;
        const int2* __restrict__ t_op_row = T.op_row;
        const uint16_t* __restrict__ t_n_parents = T.op_n_parents;
        const unsigned long long* __restrict__ t_dep_kd = T.dep_kd;
        const double* __restrict__ t_dep_rt = T.dep_rt;
        uint32_t* par_done = sv.par_done;
        const bool psm = T.par_in_smem != 0;
        const uint32_t kmask = T.kd_kmask, cmask = T.kd_cmask;
        const int csh = T.kd_cshift, fsh = T.kd_fshift, dsh = T.kd_dshift;

        // ---- init (JOB:432-484) ----
        if (psm) { for (int i = lane; i < (N + 3) / 4; i += 32) par_sm[i] = 0u; }
        else { for (int i = lane; i < N; i += 32) par_done[i] = 0u; }
        for (int i = lane; i < W; i += 32) wkey[i] = 0u;
        for (int i = lane; i < 2 * a.c_cap; i += 32) ckey0[i] = 0u;
        uint32_t* ck_cur = ckey0;             // winners among the deps of this tick's snapshot
        uint32_t* ck_nxt = ckey0 + a.c_cap;   // being built for the next tick (all zero at the start of a tick)
        OpsView ops, ops_n;
        ops.a_sm = ops_a_sm0; ops.b_sm = ops_b_sm0; ops.a_ovf = sv.ops_a_ovf[0]; ops.b_ovf = sv.ops_b_ovf[0];
        ops_n.a_sm = ops_a_sm0 + OC; ops_n.b_sm = ops_b_sm0 + OC; ops_n.a_ovf = sv.ops_a_ovf[1]; ops_n.b_ovf = sv.ops_b_ovf[1];
        for (int k = lane; k < T.n_src; k += 32) {
            const int op = __ldg(&T.src_ops[k]);
            ops_put<OC>(ops, k, __ldg(&t_op_rec[op]), __ldg(&t_op_row[op]));          // RCE:1334
        }
        __syncwarp();

        // warp-uniform state
        int nO = T.n_src;          // ready ops
        int nF = 0;                // ready flows (the frontier holds no dead entries)
        int nNF = 0;               // ready non-flow deps: zero run time (RCE:542-560), so each lives for exactly one tick
        int ops_completed = 0, deps_completed = 0;
        int tick_no = 0;
        int status = RAMP_ST_OK;
        double t = 0.0, comm = 0.0, comp = 0.0;   // lane 0: Stopwatch UT:485-496, JOB:170-171

        for (;;) {
            const bool big_ops = nO > 32 * 32;          // more op iterations per lane than win_mask has bits

            // ---- A ----
            for (int k = lane; k < nO; k += 32) {
                int4 ra; int2 rb;
                ops_get<OC>(ops, k, ra, rb);
                atomicMax(&wkey[ra.w], (uint32_t)ra.z);
            }
            __syncwarp();

            // ---- B ----
            uint32_t win_mask = 0u;
            double mo = INF;
            int na = 0;
            {
                int j = 0;
                for (int k = lane; k < nO; k += 32, ++j) {
                    int4 ra; int2 rb;
                    ops_get<OC>(ops, k, ra, rb);
                    if (wkey[ra.w] == (uint32_t)ra.z) {
                        if (j < 32) win_mask |= 1u << j;
                        ++na;
                        const double rem = __hiloint2double(ra.y, ra.x);
                        mo = (rem < mo) ? rem : mo;
                    }
                }
            }
            const double t_op = warp_min_f64(mo);
            const int n_active = warp_sum_i32(na);

            // ---- C, D: ck_cur[c] holds the arg-max key over the ready flows on channel c (built while the previous tick
            //      compacted its survivors and appended its arrivals), so the winners are the entries that match it ----
            const bool any_nf = nNF > 0;
            double t_comm = 0.0;
            if (!any_nf) {
                double md = INF;
                for (int k = lane; k < nF; k += 32) {
                    unsigned long long kd; double rem;
                    f_get<FC>(fr, k, kd, rem);
                    const uint32_t c = (uint32_t)(kd >> csh) & cmask;
                    if (c != cmask && ck_cur[c] == ((uint32_t)kd & kmask)) md = (rem < md) ? rem : md;
                }
                t_comm = warp_min_f64(md);
            }
            __syncwarp();
            // a tick that freezes the flows (any_nf) leaves the winners table as it is: its arrivals vote into ck_cur
            if (!any_nf) { for (int c = lane; c < C; c += 32) ck_cur[c] = 0u; }   // else: this table is the next tick's "next"
            uint32_t* ck_vote = any_nf ? ck_cur : ck_nxt;
            // ---- E ----
            const double tick = (t_comm < t_op) ? t_comm : t_op;

            // ---- I, J ----
            if (lane == 0) {
                const bool ticked_ops = n_active > 0;
                const bool ticked_flows = (!any_nf) && (nF > 0);                 // RCE:434-439
                if (ticked_ops && ticked_flows) { comm = __dadd_rn(comm, tick); comp = __dadd_rn(comp, tick); }
                else if (ticked_flows) comm = __dadd_rn(comm, tick);
                else if (ticked_ops) comp = __dadd_rn(comp, tick);
                t = __dadd_rn(t, tick);
                if (tick_no < a.trace_cap) { sv.tr_n[tick_no] = n_active; sv.tr_tick[tick_no] = tick; }
                else status = RAMP_ST_TRACE_OVERFLOW;
            }
            ++tick_no;

            // ---- H: the deps of the pre-tick snapshot.  A tick with ready non-flow deps is a zero-length tick that completes
            //      exactly those (RCE:412-422, 718-731) and leaves the flows untouched; any other tick ticks every flow
            //      [0, nF): survivors slide down to [0, p) and vote for the next tick's channel winners.  32 per iteration ----
            int nO_next = 0;
            int p = 0;
            if (any_nf) {
                for (int kb = 0; kb < nNF; kb += 32) {
                    const int k = kb + lane;
                    const bool valid = k < nNF;
                    uint32_t cnt = 0u, np = 1u;
                    int child = 0;
                    if (valid) {                                                                // JOB:525-536
                        const unsigned long long kd = (k < RAMP_NF_CAP) ? nf_sm[k] : nf_ovf[k - RAMP_NF_CAP];
                        child = (int)(kd >> dsh);
                        cnt = par_inc(psm, par_sm, par_done, child);                            // JOB:530
                        np = psm ? (uint32_t)(kd >> (fsh + 1)) & 0xFFu : (uint32_t)__ldg(&t_n_parents[child]);
                    }
                    const bool readied = valid && (cnt == np);                                   // JOB:531 (fires once)
                    const unsigned m = __ballot_sync(FULL, readied);
                    if (readied) ops_put_child<OC>(ops_n, nO_next + __popc(m & lt_mask), child);
                    nO_next += __popc(m);
                }
                deps_completed += nNF;
                p = nF;
                __syncwarp();
            } else {
                int ddone = 0;
                // one group of 32 flows.  FULLG: all 32 lanes hold an entry (every group but the last); INSM: the group lies in
                // the shared-memory part of the frontier (then so does everything it writes: p <= kb)
                auto h_group = [&](auto full_tag, auto insm_tag, const int kb) {
                    constexpr bool FULLG = decltype(full_tag)::value;
                    constexpr bool INSM = decltype(insm_tag)::value;
                    const int k = kb + lane;
                    const int n_here = FULLG ? 32 : ((nF - kb < 32) ? (nF - kb) : 32);
                    const bool valid = FULLG ? true : (lane < n_here);
                    unsigned long long kd = 0ull;
                    double rem = 1.0;
                    if (INSM) { if (valid) { kd = fr.kd_sm[k]; rem = fr.rem_sm[k]; } }
                    else { if (valid) f_get<FC>(fr, k, kd, rem); }
                    const double r2 = tick_down(rem, tick);                                         // JOB:561
                    const bool done = valid && (r2 == 0.0);                                         // JOB:562
                    const bool keep = valid && !done;
                    const uint32_t c = (uint32_t)(kd >> csh) & cmask;
                    if (keep && c != cmask) atomicMax(&ck_nxt[c], (uint32_t)kd & kmask);            // RCE:665-689 for the next tick
                    const unsigned dmask = __ballot_sync(FULL, done);
                    if (dmask == 0u) {
                        if (p == kb) {                                 // nothing before it died either: update in place
                            if (valid) { if (INSM) fr.rem_sm[k] = r2; else if (k < FC) fr.rem_sm[k] = r2; else fr.rem_ovf[k - FC] = r2; }
                        } else {
                            __syncwarp();                              // all lanes have read before anything is written over
                            if (valid) { if (INSM) { fr.kd_sm[p + lane] = kd; fr.rem_sm[p + lane] = r2; } else f_put<FC>(fr, p + lane, kd, r2); }
                        }
                        p += n_here;                                   // warp-uniform: every valid entry of the group survives
                    } else {
                        // JOB:525-536 for the completing lanes
                        uint32_t cnt = 0u, np = 1u;
                        int child = 0;
                        if (done) {
                            child = (int)(kd >> dsh);
                            cnt = par_inc(psm, par_sm, par_done, child);                            // JOB:530
                            np = psm ? (uint32_t)(kd >> (fsh + 1)) & 0xFFu : (uint32_t)__ldg(&t_n_parents[child]);
                        }
                        ddone += __popc(dmask);
                        const unsigned vm = FULLG ? FULL : ((1u << n_here) - 1u);
                        const unsigned mk = vm & ~dmask;
                        __syncwarp();
                        if (keep) {
                            const int q = p + __popc(mk & lt_mask);
                            if (INSM) { fr.kd_sm[q] = kd; fr.rem_sm[q] = r2; } else f_put<FC>(fr, q, kd, r2);
                        }
                        p += __popc(mk);
                        const bool readied = done && (cnt == np);                                    // JOB:531 (fires once)
                        const unsigned m = __ballot_sync(FULL, readied);
                        if (readied) ops_put_child<OC>(ops_n, nO_next + __popc(m & lt_mask), child);
                        nO_next += __popc(m);
                    }
                };
                const int n_full = nF & ~31;                           // entries covered by full groups
                const int n_full_sm = (n_full < FC) ? n_full : FC;   // FC is a multiple of 32
                int kb = 0;
                for (; kb < n_full_sm; kb += 32) h_group(std::true_type{}, std::true_type{}, kb);
                for (; kb < nF; kb += 32) h_group(std::false_type{}, std::false_type{}, kb);
                deps_completed += ddone;
            }
            // the records of the ops readied above: the first 32 are loaded here and stored after G (the loads fly while G
            // runs), any more are fetched in place
            const int n_ready = nO_next;
            __syncwarp();
            int4 rdy_a = make_int4(0, 0, 0, 0);
            int2 rdy_b = make_int2(0, 0);
            if (lane < n_ready) {
                const int child = ops_get_child<OC>(ops_n, lane);
                rdy_a = __ldg(&t_op_rec[child]);
                rdy_b = __ldg(&t_op_row[child]);
            }
            for (int k = 32 + lane; k < n_ready; k += 32) {
                const int child = ops_get_child<OC>(ops_n, k);
                ops_put<OC>(ops_n, k, __ldg(&t_op_rec[child]), __ldg(&t_op_row[child]));
            }

            // ---- G: tick the op winners; rows of the completed ops are appended at [p, tail) ----
            int tail = p;
            int nNF_next = 0;                   // this tick's non-flow arrivals (the previous ones were all consumed above)
            {
                int j = 0;
                for (int kb = 0; kb < nO; kb += 32, ++j) {
                    const int k = kb + lane;
                    const bool valid = k < nO;
                    int4 ra = make_int4(0, 0, 0, 0);
                    int2 rb = make_int2(0, 0);
                    bool done = false;
                    if (valid) {
                        ops_get<OC>(ops, k, ra, rb);
                        bool win;
                        if (big_ops) win = wkey[ra.w] == (uint32_t)ra.z;
                        else { win = ((win_mask >> j) & 1u) != 0u; wkey[ra.w] = 0u; }   // release the winner slot
                        if (win) {
                            const double rem = tick_down(__hiloint2double(ra.y, ra.x), tick);   // JOB:555
                            if (rem == 0.0) done = true;                                        // JOB:556
                            else { ra.x = __double2loint(rem); ra.y = __double2hiint(rem); }
                        }
                    }
                    const bool keep = valid && !done;
                    const unsigned km_ = __ballot_sync(FULL, keep);
                    if (keep) ops_put<OC>(ops_n, nO_next + __popc(km_ & lt_mask), ra, rb);
                    nO_next += __popc(km_);
                    const unsigned dm = __ballot_sync(FULL, done);
                    if (dm) {
                        // JOB:496-506: the out-edges of every op completed here become ready: the rows are copied as ONE
                        // flattened range so that all template loads of a batch are in flight together.
                        ops_completed += __popc(dm);
                        const int deg = done ? rb.y : 0;
                        int inc = deg;
#pragma unroll
                        for (int o = 1; o < 32; o <<= 1) {
                            const int v = __shfl_up_sync(FULL, inc, o);
                            if (lane >= o) inc += v;
                        }
                        const int total = __shfl_sync(FULL, inc, 31);
                        const int exc = inc - deg;
                        for (int jb = 0; jb < total; jb += 32 * RAMP_U) {
                            unsigned long long kd[RAMP_U];
                            double rt[RAMP_U];
#pragma unroll
                            for (int u = 0; u < RAMP_U; ++u) {
                                kd[u] = 0ull; rt[u] = 0.0;
                                if (jb + u * 32 >= total) continue;          // warp-uniform: nothing left for this slice
                                const int jf = jb + u * 32 + lane;
                                const int jc = jf < total ? jf : total - 1;
                                int lo = 0;                 // owner = first lane whose inclusive prefix exceeds jc
#pragma unroll
                                for (int step = 16; step > 0; step >>= 1) {
                                    const int v = __shfl_sync(FULL, inc, lo + step - 1);
                                    if (v <= jc) lo += step;
                                }
                                const int o_start = __shfl_sync(FULL, rb.x, lo);
                                const int o_exc = __shfl_sync(FULL, exc, lo);
                                const int e = o_start + (jc - o_exc);
                                if (jf < total) {
                                    kd[u] = __ldg(&t_dep_kd[e]);
                                    rt[u] = __ldg(&t_dep_rt[e]);                                // RCE:542-560
                                }
                            }
#pragma unroll
                            for (int u = 0; u < RAMP_U; ++u) {
                                if (jb + u * 32 >= total) continue;      // warp-uniform
                                const int jf = jb + u * 32 + lane;
                                const bool valid = jf < total;
                                const bool flow = valid && (((kd[u] >> fsh) & 1ull) != 0ull);
                                const unsigned fm = __ballot_sync(FULL, flow);
                                const unsigned nm = __ballot_sync(FULL, valid && !flow);
                                if (flow) {
                                    f_put<FC>(fr, tail + __popc(fm & lt_mask), kd[u], rt[u]);
                                    const uint32_t c = (uint32_t)(kd[u] >> csh) & cmask;
                                    if (c != cmask) atomicMax(&ck_vote[c], (uint32_t)kd[u] & kmask);
                                } else if (valid) {
                                    const int q = nNF_next + __popc(nm & lt_mask);
                                    if (q < RAMP_NF_CAP) nf_sm[q] = kd[u]; else nf_ovf[q - RAMP_NF_CAP] = kd[u];
                                }
                                tail += __popc(fm);
                                nNF_next += __popc(nm);
                            }
                        }
                    }
                }
            }
            if (lane < n_ready) ops_put<OC>(ops_n, lane, rdy_a, rdy_b);
            if (big_ops) { __syncwarp(); for (int i = lane; i < W; i += 32) wkey[i] = 0u; }
            nNF = nNF_next;
            __syncwarp();

            // ---- K, L ----
            const bool finished = (ops_completed == N) && (deps_completed == E);     // JOB:549-551
            if (!finished && isinf(tick)) status = RAMP_ST_INFINITE_TICK;             // RCE:462
            if (finished || isinf(tick)) break;
            nF = tail;
            nO = nO_next;
            { const OpsView tmp = ops; ops = ops_n; ops_n = tmp; }
            if (!any_nf) { uint32_t* tmp = ck_cur; ck_cur = ck_nxt; ck_nxt = tmp; }
        }

        // ---- results (RCE:450-452): copy the trace to an exactly-sized pool allocation ----
        const int n_rec = tick_no < a.trace_cap ? tick_no : a.trace_cap;
        long long off = -1;
        __syncwarp();
        const double steps = (double)T.num_training_steps;
        const double jct = __dmul_rn(__shfl_sync(FULL, t, 0), steps);
        const int nmw = item.n_mounted_workers > 0 ? item.n_mounted_workers : W;
        // utilisation terms go to the (now free) head of the dep-frontier overflow area
        double* term = sv.f_rem_ovf2;
        const bool can_util = (status == RAMP_ST_OK) && (tick_no <= a.trace_cap) && (n_rec <= E);
        if (can_util) util_terms(sv.tr_n, sv.tr_tick, term, n_rec, (double)nmw, jct, lane, 32);
        __syncwarp();
        if (lane == 0) {
            a.res.jct[item.slot] = jct;
            a.res.comm[item.slot] = __dmul_rn(comm, steps);
            a.res.comp[item.slot] = __dmul_rn(comp, steps);
            a.res.n_ticks[item.slot] = tick_no;
            a.res.util[item.slot] = can_util ? util_sum(term, n_rec) : 0.0;
            a.res.util_nmw[item.slot] = can_util ? nmw : -1;
            if (a.pool.top != nullptr) {
                const unsigned long long o = atomicAdd(a.pool.top, (unsigned long long)n_rec);
                if (o + (unsigned long long)n_rec <= a.pool.len) off = (long long)o;
                else if (status == RAMP_ST_OK) status = RAMP_ST_TRACE_OVERFLOW;
            }
            a.res.trace_off[item.slot] = off;
            a.res.status[item.slot] = status;
            if (a.stats) {
                atomicAdd(&a.stats->lookaheads, 1ull);
                atomicAdd(&a.stats->alg_bytes, (unsigned long long)(T.algorithmic_bytes_static + 12ull * (unsigned long long)tick_no));
            }
        }
        off = __shfl_sync(FULL, off, 0);
        __syncwarp();
        if (off >= 0) {
            for (int k = lane; k < n_rec; k += 32) {
                a.pool.n_active[off + k] = sv.tr_n[k];
                a.pool.tick[off + k] = sv.tr_tick[k];
            }
        }
        __syncwarp();
    }
}

}  // namespace ramp
#include "ramp_lookahead_cta.cuh"
#include "ramp_lookahead_thread.cuh"
namespace ramp {

// ---------------------------------------------------------------------------------------------------
// memo lookup / insert + work-list construction (RCE:469-518)

struct PlanArgs {
    const ramp_action_t* actions;   // [B]
    const TemplateDev* templates;
    int32_t n_templates;
    EpisodeState ep;
    MemoTable memo;
    WorkItem* items;                // [B] small lookaheads
    WorkItem* items_big;            // [B] big lookaheads
    WorkItem* items_res;            // [B] lookaheads on resident templates
    Counters* counters;
    MemoStats* stats;
};

__global__ void ramp_plan_kernel(const PlanArgs p) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    const int B = p.ep.B;
    if (b >= B) return;
    int32_t* ei = p.ep.ei;
    ei[EI_PLAN_SLOT * B + b] = -1;
    ei[EI_PLAN_RAN * B + b] = 0;
    const ramp_action_t act = p.actions[b];
    if ((act.flags & RAMP_ACT_SKIP) || ei[EI_DONE * B + b]) return;
    if (act.template_id < 0) return;
    if (act.template_id >= p.n_templates) {                             // the reference would KeyError on an unknown job
        atomicCAS(&p.counters->err_episode, 0, b + 1);
        ei[EI_STATUS * B + b] = RAMP_ST_BAD_TEMPLATE;
        return;
    }
    if (ei[EI_QUEUED * B + b] < 0) return;                              // reported by the step kernel
    const TemplateDev& T = p.templates[act.template_id];
    const uint32_t cap_mask = p.memo.mask;
    int slot = -1;
    bool ran = false;
    if (p.memo.mode == RAMP_MEMO_OFF) {
        slot = (int)(cap_mask + 1u) + b;
        ran = true;
    } else if (p.memo.mode == RAMP_MEMO_SHARED) {
        // level 1: the reference's per-episode memo (decides WHICH lookahead this job uses: first seen (model, degree) wins)
        const unsigned long long key = ((unsigned long long)(b + 1) << 32) | ((unsigned long long)(T.model_id & 0xFFFF) << 16)
                                       | (unsigned long long)(T.degree & 0xFFFF);
        uint32_t pos = (uint32_t)splitmix64(key) & cap_mask;
        int pos1 = -1;
        for (uint32_t probe = 0; probe <= cap_mask; ++probe) {
            const unsigned long long old = atomicCAS(&p.memo.keys[pos], 0ull, key);
            if (old == 0ull) { pos1 = (int)pos; break; }
            if (old == key) { slot = p.memo.vals[pos]; break; }          // hit RCE:495-498
            pos = (pos + 1u) & cap_mask;
        }
        atomicAdd(&p.stats->lookups, 1ull);
        if (slot >= 0) atomicAdd(&p.stats->hits, 1ull);
        else if (pos1 >= 0) {
            // level 2: has any episode of the batch already run (or claimed) the lookahead of this exact lowered job?
            const unsigned long long key2 = 0x8000000000000000ull | (unsigned long long)(T.canon_id + 1);
            uint32_t q = (uint32_t)splitmix64(key2) & p.memo.mask2;
            for (uint32_t probe = 0; probe <= p.memo.mask2; ++probe) {
                const unsigned long long old = atomicCAS(&p.memo.keys2[q], 0ull, key2);
                if (old == 0ull) { slot = p.memo.slot2_base + (int)q; ran = true; break; }
                if (old == key2) { slot = p.memo.slot2_base + (int)q; atomicAdd(&p.stats->shared_hits, 1ull); break; }
                q = (q + 1u) & p.memo.mask2;
            }
            if (slot >= 0) p.memo.vals[pos1] = slot;
        }
    } else {
        unsigned long long key;
        if (p.memo.mode == RAMP_MEMO_REFERENCE)                           // [model][max_num_partitions] per env instance RCE:491-492
            key = ((unsigned long long)(b + 1) << 32) | ((unsigned long long)(T.model_id & 0xFFFF) << 16)
                  | (unsigned long long)(T.degree & 0xFFFF);
        else
            key = 0x8000000000000000ull | (unsigned long long)(T.canon_id + 1);
        uint32_t pos = (uint32_t)splitmix64(key) & cap_mask;
        for (uint32_t probe = 0; probe <= cap_mask; ++probe) {
            const unsigned long long old = atomicCAS(&p.memo.keys[pos], 0ull, key);
            if (old == 0ull) { slot = (int)pos; ran = true; break; }      // miss: this episode runs the lookahead RCE:502-506
            if (old == key) { slot = (int)pos; break; }                   // hit RCE:495-498
            pos = (pos + 1u) & cap_mask;
        }
        // RAMP_MEMO_REFERENCE keys are per episode, so only this thread touches `pos`: vals[] holds the slot of the key's result,
        // which an overlapped step's commit kernel (ramp_commit_kernel) may have put outside the memo's own positions
        if (p.memo.mode == RAMP_MEMO_REFERENCE && slot >= 0) {
            if (ran) p.memo.vals[pos] = slot; else slot = p.memo.vals[pos];
        }
        atomicAdd(&p.stats->lookups, 1ull);
        if (slot >= 0 && !ran) atomicAdd(&p.stats->hits, 1ull);
    }
    if (slot < 0) {                                                       // table full
        atomicCAS(&p.counters->err_episode, 0, b + 1);
        ei[EI_STATUS * B + b] = RAMP_ST_TABLE_FULL;
        return;
    }
    ei[EI_PLAN_SLOT * B + b] = slot;
    ei[EI_PLAN_RAN * B + b] = ran ? 1 : 0;
    if (ran) {
        atomicAdd(&p.stats->ran, 1ull);
        WorkItem it; it.template_id = act.template_id; it.slot = slot; it.episode = b; it.n_mounted_workers = act.n_mounted_workers;
        if (T.size_class == 2) p.items_res[atomicAdd(&p.counters->n_work_res, 1)] = it;
        else if (T.size_class) p.items_big[atomicAdd(&p.counters->n_work_big, 1)] = it;
        else p.items[atomicAdd(&p.counters->n_work, 1)] = it;
    }
}

// ---------------------------------------------------------------------------------------------------
// Overlapped steps (RAMP_MEMO_REFERENCE, resident templates; DESIGN.md §4).  A lookahead's result is a function of its template
// alone, so the lookaheads of step s + 1 can run before step s has finished: the speculative plan of step s + 1 treats every
// episode with a valid, non-skip action as live and runs each (episode, template) once per reset, into a result table of its
// own.  The commit kernel then applies ramp_plan_kernel's rule exactly, in stream order, on the memo table and takes each slot
// from the result table.  An episode whose action changed after the speculative plan read it is planned again by the commit,
// into a repair table whose lookaheads run on the engine stream before the step kernel.

struct SpecRecord { int32_t flags, template_id, n_mounted_workers, slot; };   // what the speculative plan read, and its slot (-1: none)

// the result-table key: one lookahead per (episode, canonical template) between two resets
__device__ __forceinline__ unsigned long long spec_key(int b, const TemplateDev& T) {
    return ((unsigned long long)(b + 1) << 32) | (unsigned long long)(uint32_t)(T.canon_id + 1);
}

// lookup-or-insert of `key`: its position (-1: table full), *inserted when this call put it there
__device__ __forceinline__ int claim_key(unsigned long long* keys, uint32_t mask, unsigned long long key, bool* inserted) {
    uint32_t pos = (uint32_t)splitmix64(key) & mask;
    *inserted = false;
    for (uint32_t probe = 0; probe <= mask; ++probe) {
        const unsigned long long old = atomicCAS(&keys[pos], 0ull, key);
        if (old == 0ull) { *inserted = true; return (int)pos; }
        if (old == key) return (int)pos;
        pos = (pos + 1u) & mask;
    }
    return -1;
}

struct SpecPlanArgs {
    const ramp_action_t* actions;   // [B] read before the steps ahead of this one have run: a caller may still be writing it
    const TemplateDev* templates;
    int32_t n_templates, B;
    unsigned long long* keys;       // result table
    uint32_t mask;
    int32_t slot_base;              // result slot of position 0
    WorkItem* items_res;            // [B] the window's work list
    Counters* counters;             // the window's
    SpecRecord* rec;                // [B]
};

__global__ void ramp_spec_plan_kernel(const SpecPlanArgs p) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= p.B) return;
    // each field once, through volatile loads: a torn row only fails the commit's comparison
    const volatile ramp_action_t* va = p.actions + b;
    SpecRecord r;
    r.flags = va->flags; r.template_id = va->template_id; r.n_mounted_workers = va->n_mounted_workers; r.slot = -1;
    if (!(r.flags & RAMP_ACT_SKIP) && r.template_id >= 0 && r.template_id < p.n_templates) {
        const TemplateDev& T = p.templates[r.template_id];
        bool inserted = false;
        const int pos = T.size_class == 2 ? claim_key(p.keys, p.mask, spec_key(b, T), &inserted) : -1;
        if (pos >= 0) {
            r.slot = p.slot_base + pos;
            if (inserted) {
                WorkItem it; it.template_id = r.template_id; it.slot = r.slot; it.episode = b; it.n_mounted_workers = r.n_mounted_workers;
                p.items_res[atomicAdd(&p.counters->n_work_res, 1)] = it;
            }
        }
    }
    p.rec[b] = r;
}

struct CommitArgs {
    const ramp_action_t* actions;   // [B] in stream order
    const TemplateDev* templates;
    int32_t n_templates;
    EpisodeState ep;
    MemoTable memo;                 // RAMP_MEMO_REFERENCE: keys and vals
    const SpecRecord* rec;          // [B] the window's speculative plan
    unsigned long long* repair_keys;
    uint32_t repair_mask;
    int32_t repair_base;            // result slot of repair position 0
    WorkItem* items_res;            // [B] repair work list (the window's, its lookaheads have finished)
    Counters* win_counters;
    Counters* counters;             // the engine's: err_episode
    MemoStats* stats;
};

// ramp_plan_kernel's rule for RAMP_MEMO_REFERENCE, statement for statement, except where the slot comes from
__global__ void ramp_commit_kernel(const CommitArgs p) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    const int B = p.ep.B;
    if (b >= B) return;
    int32_t* ei = p.ep.ei;
    ei[EI_PLAN_SLOT * B + b] = -1;
    ei[EI_PLAN_RAN * B + b] = 0;
    const ramp_action_t act = p.actions[b];
    if ((act.flags & RAMP_ACT_SKIP) || ei[EI_DONE * B + b]) return;
    if (act.template_id < 0) return;
    if (act.template_id >= p.n_templates) {
        atomicCAS(&p.counters->err_episode, 0, b + 1);
        ei[EI_STATUS * B + b] = RAMP_ST_BAD_TEMPLATE;
        return;
    }
    if (ei[EI_QUEUED * B + b] < 0) return;
    const TemplateDev& T = p.templates[act.template_id];
    const uint32_t cap_mask = p.memo.mask;
    const unsigned long long key = ((unsigned long long)(b + 1) << 32) | ((unsigned long long)(T.model_id & 0xFFFF) << 16)
                                   | (unsigned long long)(T.degree & 0xFFFF);
    bool ran = false;
    const int pos = claim_key(p.memo.keys, cap_mask, key, &ran);
    atomicAdd(&p.stats->lookups, 1ull);
    if (pos >= 0 && !ran) atomicAdd(&p.stats->hits, 1ull);
    int slot = -1;
    if (pos >= 0) {
        if (!ran) slot = p.memo.vals[pos];
        else {
            const SpecRecord r = p.rec[b];
            if (r.slot >= 0 && r.flags == act.flags && r.template_id == act.template_id && r.n_mounted_workers == act.n_mounted_workers) {
                slot = r.slot;
            } else {
                bool inserted = false;
                const int q = claim_key(p.repair_keys, p.repair_mask, spec_key(b, T), &inserted);
                if (q >= 0) {
                    slot = p.repair_base + q;
                    if (inserted) {
                        WorkItem it; it.template_id = act.template_id; it.slot = slot; it.episode = b; it.n_mounted_workers = act.n_mounted_workers;
                        p.items_res[atomicAdd(&p.win_counters->n_work_res, 1)] = it;
                    }
                }
            }
            if (slot >= 0) p.memo.vals[pos] = slot;
        }
    }
    if (slot < 0) {
        atomicCAS(&p.counters->err_episode, 0, b + 1);
        ei[EI_STATUS * B + b] = RAMP_ST_TABLE_FULL;
        return;
    }
    ei[EI_PLAN_SLOT * B + b] = slot;
    ei[EI_PLAN_RAN * B + b] = ran ? 1 : 0;
    if (ran) atomicAdd(&p.stats->ran, 1ull);
}

// ---------------------------------------------------------------------------------------------------
// RampClusterEnvironment.step (RCE:894-1179): one thread per episode; serial f64 in the reference's order.

struct StepArgs {
    const ramp_action_t* actions;   // [B]
    EpisodeState ep;
    ResultSlots res;
    TracePool pool;
    Counters* counters;
    double* stats_out;              // [B][RAMP_STEP_STATS_LEN] or null
    int32_t* n_cluster_steps_out;   // [B] or null
    int32_t fuse_empty_steps;
};

#define EF(f) ef[(f) * B + b]
#define EI(f) ei[(f) * B + b]

// One episode's scalars and running-job table, wherever they live: field f of the scalars at ef[f * ld], row `row` of the table
// at rf[(f * rows + row) * ld].  The HBM arrays of EpisodeState are the view {ep.ef + b, ..., ld = B, rows = max_running}; the step
// kernel runs on a copy in shared memory, {.. + threadIdx.x, ld = CTA threads, rows = step_rows}
struct EpView {
    double* ef; int32_t* ei; double* rf; int32_t* ri;
    int ld, rows;
};
#define VF(f) v.ef[(f) * v.ld]
#define VI(f) v.ei[(f) * v.ld]
#define VRF(f, row) v.rf[((f) * v.rows + (row)) * v.ld]
#define VRI(f, row) v.ri[((f) * v.rows + (row)) * v.ld]

__device__ __forceinline__ EpView hbm_view(const EpisodeState& ep, int b) {
    EpView v;
    v.ef = ep.ef + b; v.ei = ep.ei + b; v.rf = ep.rf + b; v.ri = ep.ri + b; v.ld = ep.B; v.rows = ep.max_running;
    return v;
}

// rows of the running-job table the step kernel keeps on chip: at most max_jobs jobs of an episode ever run
__host__ __device__ inline int step_rows(int max_running, int max_jobs) { return max_running < max_jobs ? max_running : max_jobs; }
// shared memory of a step-kernel CTA of nt threads (one per episode)
__host__ __device__ inline size_t step_smem_bytes(int nt, int rows) {
    return (size_t)nt * ((size_t)(EF_COUNT + RF_COUNT * rows) * 8 + (size_t)(EI_COUNT + RI_COUNT * rows) * 4);
}

__device__ __forceinline__ void step_register_blocked(const EpisodeState& ep, const EpView& v, int b, int job_idx, double* st) {   // RCE:1504-1540
    ramp_job_record_t& r = ep.rec[(size_t)b * ep.max_jobs + job_idx];
    if (VI(EI_QUEUED) == job_idx) VI(EI_QUEUED) = -1;
    if (r.status == RAMP_JS_BLOCKED) return;
    r.status = RAMP_JS_BLOCKED;
    r.event_seq = VI(EI_EVENT_SEQ)++;
    VI(EI_NUM_BLOCKED)++;
    st[RAMP_SS_NUM_JOBS_BLOCKED] += 1.0;
}

__device__ __forceinline__ void step_remove_running(const EpView& v, int pos) {   // keeps dict (insertion) order
    const int n = VI(EI_N_RUNNING);
    for (int k = pos; k + 1 < n; ++k) {
        for (int f = 0; f < RF_COUNT; ++f) VRF(f, k) = VRF(f, k + 1);
        for (int f = 0; f < RI_COUNT; ++f) VRI(f, k) = VRI(f, k + 1);
    }
    VI(EI_N_RUNNING) = n - 1;
}

// n_jobs: ep.n_jobs_ep[b]
__device__ __forceinline__ bool step_is_done(const EpisodeState& ep, const EpView& v, int n_jobs) {   // RCE:1542-1557
    if (VF(EF_NOW) >= ep.max_sim_time) return true;
    return (n_jobs - VI(EI_NUM_ARRIVED)) <= 0 && VI(EI_N_RUNNING) == 0 && VI(EI_QUEUED) < 0;
}

__device__ __forceinline__ void step_get_next_job(const EpisodeState& ep, const EpView& v, int b) {   // RCE:351-377
    const int k = VI(EI_NUM_ARRIVED);
    ramp_job_record_t& r = ep.rec[(size_t)b * ep.max_jobs + k];
    r.status = RAMP_JS_QUEUED; r.event_seq = 0;
    r.time_arrived = VF(EF_NOW); r.time_started = 0.0; r.time_completed = 0.0;
    r.jct = r.comm = r.comp = r.util = 0.0;
    const ramp_arrival_t a = ep.arr[(size_t)b * ep.max_jobs + k];
    VF(EF_LAST_ARRIVAL) = VF(EF_NOW);                                        // RCE:362
    VF(EF_NEXT_ARRIVAL) = __dadd_rn(VF(EF_NEXT_ARRIVAL), a.interarrival);    // RCE:363
    VF(EF_LOAD_SUM) = __dadd_rn(VF(EF_LOAD_SUM),
                                __ddiv_rn(__dadd_rn(a.orig_op_mem, a.orig_dep_size),
                                          __dsub_rn(VF(EF_NEXT_ARRIVAL), VF(EF_LAST_ARRIVAL))));   // RCE:364
    VI(EI_LOAD_N)++;
    VI(EI_NUM_ARRIVED) = k + 1;
}

// One thread per episode, NT per CTA.  Three parts:
//   prologue  the episode's scalars and the live rows of its running-job table are copied from HBM into shared memory in one batch
//             of independent loads;
//   body      the cluster steps on the on-chip copy: the same f64 operations in the same order as on HBM.  Job records, arrivals,
//             result slots, traces, es rows and the outputs stay in HBM;
//   epilogue  the scalars and every table row the body may have written go back to HBM, so every other kernel sees the layout
//             and the values it always saw.
template <int NT>
__global__ void __launch_bounds__(NT) ramp_step_kernel(const StepArgs s) {
    extern __shared__ __align__(16) unsigned char step_smem[];
    const int b = blockIdx.x * NT + threadIdx.x;
    const EpisodeState& ep = s.ep;
    const int B = ep.B, R = ep.max_running;
    if (b >= B) return;
    const int rows = step_rows(R, ep.max_jobs);
    EpView v;
    v.ld = NT; v.rows = rows;
    v.ef = reinterpret_cast<double*>(step_smem) + threadIdx.x;                    // [EF_COUNT][NT]
    v.rf = reinterpret_cast<double*>(step_smem) + EF_COUNT * NT + threadIdx.x;    // [RF_COUNT][rows][NT]
    v.ei = reinterpret_cast<int32_t*>(reinterpret_cast<double*>(step_smem) + (EF_COUNT + RF_COUNT * rows) * NT) + threadIdx.x;   // [EI_COUNT][NT]
    v.ri = v.ei + EI_COUNT * NT;                                                   // [RI_COUNT][rows][NT]
    const EpView h = hbm_view(ep, b);

    // ---- prologue ----
    {
        double f64[EF_COUNT];
        int32_t i32[EI_COUNT];
#pragma unroll
        for (int f = 0; f < EF_COUNT; ++f) f64[f] = h.ef[f * h.ld];
#pragma unroll
        for (int f = 0; f < EI_COUNT; ++f) i32[f] = h.ei[f * h.ld];
#pragma unroll
        for (int f = 0; f < EF_COUNT; ++f) VF(f) = f64[f];
#pragma unroll
        for (int f = 0; f < EI_COUNT; ++f) VI(f) = i32[f];
        const int n0 = i32[EI_N_RUNNING];
        for (int k = 0; k < n0; ++k) {
            double rf64[RF_COUNT];
            int32_t ri32[RI_COUNT];
#pragma unroll
            for (int f = 0; f < RF_COUNT; ++f) rf64[f] = h.rf[(f * h.rows + k) * h.ld];
#pragma unroll
            for (int f = 0; f < RI_COUNT; ++f) ri32[f] = h.ri[(f * h.rows + k) * h.ld];
#pragma unroll
            for (int f = 0; f < RF_COUNT; ++f) VRF(f, k) = rf64[f];
#pragma unroll
            for (int f = 0; f < RI_COUNT; ++f) VRI(f, k) = ri32[f];
        }
    }
    const int n_jobs = ep.n_jobs_ep[b];
    const ramp_action_t act = s.actions[b];
    int hi_row = VI(EI_N_RUNNING);          // rows [0, hi_row) may differ from HBM at the end

    double st[RAMP_STEP_STATS_LEN];
    double st0[RAMP_STEP_STATS_LEN];
#pragma unroll
    for (int k = 0; k < RAMP_STEP_STATS_LEN; ++k) { st[k] = 0.0; st0[k] = 0.0; }
    int n_cluster_steps = 0;

    if (!((act.flags & RAMP_ACT_SKIP) || VI(EI_DONE))) {
        for (int cs = 0;; ++cs) {
#pragma unroll
            for (int k = 0; k < RAMP_STEP_STATS_LEN; ++k) st[k] = 0.0;
            st[RAMP_SS_STEP_COUNTER] = (double)VI(EI_STEP_COUNTER);            // RCE:309
            st[RAMP_SS_STEP_START_TIME] = VF(EF_NOW);                          // RCE:310
            bool has_action = (cs == 0) && act.template_id >= 0;
            int handled = -1;
            if (has_action) {
                handled = VI(EI_QUEUED);
                if (handled < 0 || VI(EI_PLAN_SLOT) < 0) {
                    if (handled < 0) { VI(EI_STATUS) = RAMP_ST_NO_QUEUED_JOB; atomicCAS(&s.counters->err_episode, 0, b + 1); }
                    has_action = false;
                }
            }
            // RCE:914-919: queued jobs not handled by the action are blocked
            if (!has_action && VI(EI_QUEUED) >= 0) step_register_blocked(ep, v, b, VI(EI_QUEUED), st);

            if (has_action) {
                const int slot = VI(EI_PLAN_SLOT);
                VI(EI_LAST_SLOT) = slot;
                st[RAMP_SS_LOOKAHEAD_RAN] = (double)VI(EI_PLAN_RAN);
                ramp_job_record_t& r = ep.rec[(size_t)b * ep.max_jobs + handled];
                r.status = RAMP_JS_RUNNING;
                r.time_started = VF(EF_NOW);                                    // RCE:1418
                VI(EI_QUEUED) = -1;                                             // RCE:1420
                const int lst = s.res.status[slot];
                if (lst != RAMP_ST_OK) {                                        // the reference raises (RCE:462)
                    VI(EI_STATUS) = lst; atomicCAS(&s.counters->err_episode, 0, b + 1);
                    step_register_blocked(ep, v, b, handled, st);
                } else {
                    const double jct = s.res.jct[slot];
                    if (jct > act.max_acceptable_jct) {                         // RCE:815 (strict)
                        step_register_blocked(ep, v, b, handled, st);              // RCE:821-824
                    } else if (VI(EI_N_RUNNING) >= R) {
                        VI(EI_STATUS) = RAMP_ST_TABLE_FULL; atomicCAS(&s.counters->err_episode, 0, b + 1);
                        step_register_blocked(ep, v, b, handled, st);
                    } else {
                        // RCE:830-832: computed by the lookahead kernel for its own mounted-worker count; a memo hit from a job
                        // mounted on a different number of workers recomputes it here (serial sum in tick order)
                        double util = 0.0;
                        if (s.res.util_nmw[slot] == act.n_mounted_workers) {
                            util = s.res.util[slot];
                        } else {
                            const long long off = s.res.trace_off[slot];
                            const int T = s.res.n_ticks[slot];
                            const double nmw = (double)act.n_mounted_workers;
                            if (off >= 0) {
                                for (int k = 0; k < T; ++k)
                                    util = __dadd_rn(util, __dmul_rn(__ddiv_rn((double)s.pool.n_active[off + k], nmw),
                                                                     __ddiv_rn(s.pool.tick[off + k], jct)));
                            }
                        }
                        const int row = VI(EI_N_RUNNING)++;
                        if (row >= hi_row) hi_row = row + 1;
                        const ramp_arrival_t arr = ep.arr[(size_t)b * ep.max_jobs + handled];
                        VRF(RF_JCT, row) = jct; VRF(RF_STARTED, row) = VF(EF_NOW);
                        VRF(RF_COMM_FRAC, row) = __ddiv_rn(s.res.comm[slot], jct); VRF(RF_COMP_FRAC, row) = __ddiv_rn(s.res.comp[slot], jct);
                        VRF(RF_UTIL, row) = util;
                        VRF(RF_PART_OP_MEM, row) = act.part_op_mem; VRF(RF_PART_DEP, row) = act.part_dep_size;
                        VRF(RF_FLOW, row) = act.flow_size;
                        VRF(RF_ORIG_OP_MEM, row) = arr.orig_op_mem; VRF(RF_ORIG_DEP, row) = arr.orig_dep_size;
                        VRI(RI_JOB_IDX, row) = handled; VRI(RI_N_WORKERS, row) = act.n_mounted_workers;
                        VRI(RI_N_CHANNELS, row) = act.n_mounted_channels;
                        r.jct = jct; r.comm = s.res.comm[slot]; r.comp = s.res.comp[slot]; r.util = util;
                    }
                }
            }

            // ---- outer event loop RCE:942-1044 ----
            double util_mounted_sum = 0.0, util_cluster_sum = 0.0;
            double sum_jobs = 0.0, sum_workers = 0.0, sum_channels = 0.0, sum_comp_frac = 0.0, sum_comm_frac = 0.0;
            int n_frac = 0, n_iter = 0;
            bool step_done = false;
            while (!step_done) {
                const double now = VF(EF_NOW);
                double tick = __dsub_rn(VF(EF_NEXT_ARRIVAL), now);                           // RCE:950
                { const double b2 = __dsub_rn(ep.max_sim_time, now); if (b2 < tick) tick = b2; }
                const int nr = VI(EI_N_RUNNING);
                for (int k = 0; k < nr; ++k) {                                               // RCE:951-954
                    const double remaining = __dsub_rn(VRF(RF_JCT, k), __dsub_rn(now, VRF(RF_STARTED, k)));
                    if (remaining < tick) tick = remaining;
                }
                int mounted_workers = 0, mounted_channels = 0;
                double util_sum = 0.0;
                for (int k = 0; k < nr; ++k) {                                               // RCE:962-982
                    const double jct = VRF(RF_JCT, k);
                    const double frac = __ddiv_rn(tick, jct);
                    const double pom = VRF(RF_PART_OP_MEM, k), pds = VRF(RF_PART_DEP, k);
                    const double oom = VRF(RF_ORIG_OP_MEM, k), ods = VRF(RF_ORIG_DEP, k);
                    st[RAMP_SS_COMPUTE_INFO_PROCESSED] = __dadd_rn(st[RAMP_SS_COMPUTE_INFO_PROCESSED], __dmul_rn(pom, frac));
                    st[RAMP_SS_DEP_INFO_PROCESSED] = __dadd_rn(st[RAMP_SS_DEP_INFO_PROCESSED], __dmul_rn(pds, frac));
                    st[RAMP_SS_FLOW_INFO_PROCESSED] = __dadd_rn(st[RAMP_SS_FLOW_INFO_PROCESSED], __dmul_rn(VRF(RF_FLOW, k), frac));
                    st[RAMP_SS_CLUSTER_INFO_PROCESSED] = __dadd_rn(st[RAMP_SS_CLUSTER_INFO_PROCESSED], __dmul_rn(__dadd_rn(pom, pds), frac));
                    st[RAMP_SS_DEMAND_COMPUTE_INFO_PROCESSED] = __dadd_rn(st[RAMP_SS_DEMAND_COMPUTE_INFO_PROCESSED], __dmul_rn(oom, frac));
                    st[RAMP_SS_DEMAND_DEP_INFO_PROCESSED] = __dadd_rn(st[RAMP_SS_DEMAND_DEP_INFO_PROCESSED], __dmul_rn(ods, frac));
                    st[RAMP_SS_DEMAND_TOTAL_INFO_PROCESSED] = __dadd_rn(st[RAMP_SS_DEMAND_TOTAL_INFO_PROCESSED], __dmul_rn(__dadd_rn(oom, ods), frac));
                    sum_comp_frac = __dadd_rn(sum_comp_frac, VRF(RF_COMP_FRAC, k));
                    sum_comm_frac = __dadd_rn(sum_comm_frac, VRF(RF_COMM_FRAC, k));
                    ++n_frac;
                    mounted_workers += VRI(RI_N_WORKERS, k);      // workers / channels of distinct jobs are disjoint (ramp_rules.py:1-40)
                    mounted_channels += VRI(RI_N_CHANNELS, k);
                    util_sum = __dadd_rn(util_sum, VRF(RF_UTIL, k));
                }
                sum_jobs = __dadd_rn(sum_jobs, (double)nr);                                   // RCE:984
                sum_workers = __dadd_rn(sum_workers, (double)mounted_workers);               // RCE:986
                sum_channels = __dadd_rn(sum_channels, (double)mounted_channels);            // RCE:987
                double tick_mounted = 0.0, tick_cluster = 0.0;
                if (nr > 0) {                                                                // RCE:989-994
                    tick_mounted = __ddiv_rn(util_sum, (double)nr);
                    tick_cluster = __dmul_rn(__ddiv_rn((double)mounted_workers, (double)ep.n_cluster_workers), tick_mounted);
                    util_mounted_sum = __dadd_rn(util_mounted_sum, tick_mounted);
                    util_cluster_sum = __dadd_rn(util_cluster_sum, tick_cluster);
                }
                if (ep.tick_util && n_iter < ep.tick_util_cap) {
                    double* tu = ep.tick_util + ((size_t)b * ep.tick_util_cap + n_iter) * 2;
                    tu[0] = tick_mounted; tu[1] = tick_cluster;
                }
                ++n_iter;
                VF(EF_NOW) = __dadd_rn(now, tick);                                            // RCE:998
                const double now2 = VF(EF_NOW);

                // RCE:1004-1017, 1466-1502
                int k = 0;
                while (k < VI(EI_N_RUNNING)) {
                    const double remaining = __dsub_rn(__dsub_rn(VRF(RF_JCT, k), __dsub_rn(now2, VRF(RF_STARTED, k))), ep.eps);
                    if (remaining <= 0.0) {
                        ramp_job_record_t& r = ep.rec[(size_t)b * ep.max_jobs + VRI(RI_JOB_IDX, k)];
                        r.status = RAMP_JS_COMPLETED; r.time_completed = now2;
                        r.event_seq = VI(EI_EVENT_SEQ)++;
                        VI(EI_NUM_COMPLETED)++;
                        st[RAMP_SS_NUM_JOBS_COMPLETED] += 1.0;
                        step_remove_running(v, k);
                        step_done = true;
                    } else {
                        ++k;
                    }
                }
                // RCE:1019-1040
                if ((n_jobs - VI(EI_NUM_ARRIVED)) > 0) {
                    if (__dadd_rn(now2, ep.eps) >= VF(EF_NEXT_ARRIVAL)) {
                        const int idx = VI(EI_NUM_ARRIVED);
                        step_get_next_job(ep, v, b);
                        st[RAMP_SS_NUM_JOBS_ARRIVED] += 1.0;
                        if (VI(EI_QUEUED) < 0 && ep.queue_capacity >= 1) VI(EI_QUEUED) = idx;   // RCE:1030-1031
                        else step_register_blocked(ep, v, b, idx, st);                             // RCE:1034
                        step_done = true;
                    }
                } else {
                    VF(EF_NEXT_ARRIVAL) = __longlong_as_double(RAMP_INF_BITS);                  // RCE:1040
                }
                if (step_is_done(ep, v, n_jobs)) step_done = true;                                       // RCE:1043
            }

            // ---- RCE:1046-1084 ----
            st[RAMP_SS_STEP_END_TIME] = VF(EF_NOW);
            st[RAMP_SS_STEP_TIME] = __dsub_rn(st[RAMP_SS_STEP_END_TIME], st[RAMP_SS_STEP_START_TIME]);
            st[RAMP_SS_MEAN_NUM_JOBS_RUNNING] = __ddiv_rn(sum_jobs, (double)n_iter);
            st[RAMP_SS_MEAN_NUM_MOUNTED_WORKERS] = __ddiv_rn(sum_workers, (double)n_iter);
            st[RAMP_SS_MEAN_NUM_MOUNTED_CHANNELS] = __ddiv_rn(sum_channels, (double)n_iter);
            st[RAMP_SS_MEAN_COMPUTE_OVERHEAD_FRAC] = n_frac > 0 ? __ddiv_rn(sum_comp_frac, (double)n_frac) : 0.0;
            st[RAMP_SS_MEAN_COMMUNICATION_OVERHEAD_FRAC] = n_frac > 0 ? __ddiv_rn(sum_comm_frac, (double)n_frac) : 0.0;
            {
                const double dt = st[RAMP_SS_STEP_TIME];
#define RAMP_TP(dst, src) st[dst] = (st[src] != 0.0 && dt != 0.0) ? __ddiv_rn(st[src], dt) : 0.0   /* RCE:1064-1077 */
                RAMP_TP(RAMP_SS_MEAN_COMPUTE_THROUGHPUT, RAMP_SS_COMPUTE_INFO_PROCESSED);
                RAMP_TP(RAMP_SS_MEAN_DEP_THROUGHPUT, RAMP_SS_DEP_INFO_PROCESSED);
                RAMP_TP(RAMP_SS_MEAN_FLOW_THROUGHPUT, RAMP_SS_FLOW_INFO_PROCESSED);
                RAMP_TP(RAMP_SS_MEAN_CLUSTER_THROUGHPUT, RAMP_SS_CLUSTER_INFO_PROCESSED);
                RAMP_TP(RAMP_SS_MEAN_DEMAND_COMPUTE_THROUGHPUT, RAMP_SS_DEMAND_COMPUTE_INFO_PROCESSED);
                RAMP_TP(RAMP_SS_MEAN_DEMAND_DEP_THROUGHPUT, RAMP_SS_DEMAND_DEP_INFO_PROCESSED);
                RAMP_TP(RAMP_SS_MEAN_DEMAND_TOTAL_THROUGHPUT, RAMP_SS_DEMAND_TOTAL_INFO_PROCESSED);
#undef RAMP_TP
            }
            st[RAMP_SS_UTIL_MOUNTED_SUM] = util_mounted_sum;
            st[RAMP_SS_UTIL_CLUSTER_SUM] = util_cluster_sum;
            st[RAMP_SS_NUM_TICKS] = (double)n_iter;
            if (ep.tick_util) ep.tick_util_n[b] = n_iter;
            st[RAMP_SS_JOB_QUEUE_LENGTH] = VI(EI_QUEUED) >= 0 ? 1.0 : 0.0;                       // RCE:1082
            if (s.ep.es) {
                // eval_loop.py:50-97: this cluster step into the env-step's row, in cluster-step order; the action step (cs 0) opens
                // it.  The end-of-episode blocks below come after RCE:1084 logged the step, so they are not in it
                double* es = s.ep.es + (size_t)b * ES_STRIDE;
                const bool open = cs == 0;
#define RAMP_ES_ADD(e, src) es[e] = __dadd_rn(open ? 0.0 : es[e], st[src])
                es[RAMP_ESS_STEP_COUNTER] = st[RAMP_SS_STEP_COUNTER];                               // eval_loop.py:96-97 last
                if (open) es[RAMP_ESS_STEP_START_TIME] = st[RAMP_SS_STEP_START_TIME];                   // :66-68 first
                es[RAMP_ESS_STEP_END_TIME] = st[RAMP_SS_STEP_END_TIME];                             // :70-72 last
                RAMP_ES_ADD(RAMP_ESS_MEAN_NUM_MOUNTED_WORKERS, RAMP_SS_MEAN_NUM_MOUNTED_WORKERS);            // :74-83 'mean': sum here,
                RAMP_ES_ADD(RAMP_ESS_MEAN_NUM_MOUNTED_CHANNELS, RAMP_SS_MEAN_NUM_MOUNTED_CHANNELS);          //   / cluster steps at the end
                RAMP_ES_ADD(RAMP_ESS_MEAN_COMPUTE_THROUGHPUT, RAMP_SS_MEAN_COMPUTE_THROUGHPUT);
                RAMP_ES_ADD(RAMP_ESS_MEAN_DEP_THROUGHPUT, RAMP_SS_MEAN_DEP_THROUGHPUT);
                RAMP_ES_ADD(RAMP_ESS_MEAN_CLUSTER_THROUGHPUT, RAMP_SS_MEAN_CLUSTER_THROUGHPUT);
                RAMP_ES_ADD(RAMP_ESS_MEAN_DEMAND_COMPUTE_THROUGHPUT, RAMP_SS_MEAN_DEMAND_COMPUTE_THROUGHPUT);
                RAMP_ES_ADD(RAMP_ESS_MEAN_DEMAND_DEP_THROUGHPUT, RAMP_SS_MEAN_DEMAND_DEP_THROUGHPUT);
                RAMP_ES_ADD(RAMP_ESS_MEAN_DEMAND_TOTAL_THROUGHPUT, RAMP_SS_MEAN_DEMAND_TOTAL_THROUGHPUT);
                RAMP_ES_ADD(RAMP_ESS_MEAN_COMPUTE_OVERHEAD_FRAC, RAMP_SS_MEAN_COMPUTE_OVERHEAD_FRAC);
                RAMP_ES_ADD(RAMP_ESS_MEAN_COMMUNICATION_OVERHEAD_FRAC, RAMP_SS_MEAN_COMMUNICATION_OVERHEAD_FRAC);
                RAMP_ES_ADD(RAMP_ESS_MEAN_NUM_JOBS_RUNNING, RAMP_SS_MEAN_NUM_JOBS_RUNNING);
                RAMP_ES_ADD(RAMP_ESS_MEAN_FLOW_THROUGHPUT, RAMP_SS_MEAN_FLOW_THROUGHPUT);
                RAMP_ES_ADD(RAMP_ESS_NUM_JOBS_COMPLETED, RAMP_SS_NUM_JOBS_COMPLETED);                    // :85-94 the rest: np.sum
                RAMP_ES_ADD(RAMP_ESS_NUM_JOBS_ARRIVED, RAMP_SS_NUM_JOBS_ARRIVED);
                RAMP_ES_ADD(RAMP_ESS_NUM_JOBS_BLOCKED, RAMP_SS_NUM_JOBS_BLOCKED);
#pragma unroll
                for (int k = 0; k < 7; ++k) RAMP_ES_ADD(RAMP_ESS_COMPUTE_INFO_PROCESSED + k, RAMP_SS_COMPUTE_INFO_PROCESSED + k);
                RAMP_ES_ADD(RAMP_ESS_STEP_TIME, RAMP_SS_STEP_TIME);
                RAMP_ES_ADD(RAMP_ESS_JOB_QUEUE_LENGTH, RAMP_SS_JOB_QUEUE_LENGTH);
                RAMP_ES_ADD(RAMP_ESS_MEAN_MOUNTED_WORKER_UTILISATION_FRAC, RAMP_SS_UTIL_MOUNTED_SUM);        // per-tick lists: sums
                RAMP_ES_ADD(RAMP_ESS_MEAN_CLUSTER_WORKER_UTILISATION_FRAC, RAMP_SS_UTIL_CLUSTER_SUM);        //   and their length
                RAMP_ES_ADD(ES_TICKS, RAMP_SS_NUM_TICKS);
#undef RAMP_ES_ADD
            }
            // RCE:1086-1106: this cluster step's contribution to episode_stats
#pragma unroll
            for (int k = 0; k < 7; ++k) VF(EF_ACC_INFO + k) = __dadd_rn(VF(EF_ACC_INFO + k), st[RAMP_SS_COMPUTE_INFO_PROCESSED + k]);
            VF(EF_ACC_COMP_FRAC) = __dadd_rn(VF(EF_ACC_COMP_FRAC), st[RAMP_SS_MEAN_COMPUTE_OVERHEAD_FRAC]);
            VF(EF_ACC_COMM_FRAC) = __dadd_rn(VF(EF_ACC_COMM_FRAC), st[RAMP_SS_MEAN_COMMUNICATION_OVERHEAD_FRAC]);
            VF(EF_ACC_JOBS_RUNNING) = __dadd_rn(VF(EF_ACC_JOBS_RUNNING), st[RAMP_SS_MEAN_NUM_JOBS_RUNNING]);
            VF(EF_ACC_MOUNTED_WORKERS) = __dadd_rn(VF(EF_ACC_MOUNTED_WORKERS), st[RAMP_SS_MEAN_NUM_MOUNTED_WORKERS]);
            VF(EF_ACC_UTIL_MOUNTED) = __dadd_rn(VF(EF_ACC_UTIL_MOUNTED), st[RAMP_SS_UTIL_MOUNTED_SUM]);
            VF(EF_ACC_UTIL_CLUSTER) = __dadd_rn(VF(EF_ACC_UTIL_CLUSTER), st[RAMP_SS_UTIL_CLUSTER_SUM]);
            VF(EF_ACC_TICKS) = __dadd_rn(VF(EF_ACC_TICKS), st[RAMP_SS_NUM_TICKS]);
            VF(EF_ACC_STEPS) = __dadd_rn(VF(EF_ACC_STEPS), 1.0);
            VI(EI_STEP_COUNTER)++;                                                                // RCE:1109
            const bool done = step_is_done(ep, v, n_jobs);
            if (done) {                                                                           // RCE:1111-1121
                while (VI(EI_N_RUNNING) > 0) {
                    step_register_blocked(ep, v, b, VRI(RI_JOB_IDX, 0), st);
                    step_remove_running(v, 0);
                }
                VI(EI_DONE) = 1;
            }
            st[RAMP_SS_DONE] = done ? 1.0 : 0.0;
            ++n_cluster_steps;
            if (cs == 0) {
#pragma unroll
                for (int k = 0; k < RAMP_STEP_STATS_LEN; ++k) st0[k] = st[k];
            }
            // RJPE:394-395: while len(job_queue) == 0 and not is_done(): step(Action())
            if (!s.fuse_empty_steps || done || VI(EI_QUEUED) >= 0) break;
        }
        if (s.ep.es) {
            // the env-step ends: its row (eval_loop.py:74-83).  np.mean over the cluster steps is their sum (in order) / their number;
            // the per-tick lists' mean is over every entry of the env-step
            double* es = s.ep.es + (size_t)b * ES_STRIDE;
            const double n = (double)n_cluster_steps;
#define RAMP_ES_MEAN(e) es[e] = __ddiv_rn(es[e], n)
            RAMP_ES_MEAN(RAMP_ESS_MEAN_NUM_MOUNTED_WORKERS); RAMP_ES_MEAN(RAMP_ESS_MEAN_NUM_MOUNTED_CHANNELS);
            RAMP_ES_MEAN(RAMP_ESS_MEAN_COMPUTE_THROUGHPUT); RAMP_ES_MEAN(RAMP_ESS_MEAN_DEP_THROUGHPUT);
            RAMP_ES_MEAN(RAMP_ESS_MEAN_CLUSTER_THROUGHPUT); RAMP_ES_MEAN(RAMP_ESS_MEAN_DEMAND_COMPUTE_THROUGHPUT);
            RAMP_ES_MEAN(RAMP_ESS_MEAN_DEMAND_DEP_THROUGHPUT); RAMP_ES_MEAN(RAMP_ESS_MEAN_DEMAND_TOTAL_THROUGHPUT);
            RAMP_ES_MEAN(RAMP_ESS_MEAN_COMPUTE_OVERHEAD_FRAC); RAMP_ES_MEAN(RAMP_ESS_MEAN_COMMUNICATION_OVERHEAD_FRAC);
            RAMP_ES_MEAN(RAMP_ESS_MEAN_NUM_JOBS_RUNNING); RAMP_ES_MEAN(RAMP_ESS_MEAN_FLOW_THROUGHPUT);
#undef RAMP_ES_MEAN
            const double ticks = es[ES_TICKS];                     // >= 1: every cluster step ticks at least once
            es[RAMP_ESS_MEAN_MOUNTED_WORKER_UTILISATION_FRAC] = __ddiv_rn(es[RAMP_ESS_MEAN_MOUNTED_WORKER_UTILISATION_FRAC], ticks);
            es[RAMP_ESS_MEAN_CLUSTER_WORKER_UTILISATION_FRAC] = __ddiv_rn(es[RAMP_ESS_MEAN_CLUSTER_WORKER_UTILISATION_FRAC], ticks);
        }
        if (s.fuse_empty_steps) st0[RAMP_SS_DONE] = VI(EI_DONE) ? 1.0 : 0.0;
    } else {
        st0[RAMP_SS_DONE] = VI(EI_DONE) ? 1.0 : 0.0;
        st0[RAMP_SS_STEP_COUNTER] = (double)VI(EI_STEP_COUNTER);
        st0[RAMP_SS_JOB_QUEUE_LENGTH] = VI(EI_QUEUED) >= 0 ? 1.0 : 0.0;
    }

    // ---- epilogue ----
#pragma unroll
    for (int f = 0; f < EF_COUNT; ++f) h.ef[f * h.ld] = VF(f);
#pragma unroll
    for (int f = 0; f < EI_COUNT; ++f) h.ei[f * h.ld] = VI(f);
    for (int k = 0; k < hi_row; ++k) {
#pragma unroll
        for (int f = 0; f < RF_COUNT; ++f) h.rf[(f * h.rows + k) * h.ld] = VRF(f, k);
#pragma unroll
        for (int f = 0; f < RI_COUNT; ++f) h.ri[(f * h.rows + k) * h.ld] = VRI(f, k);
    }
    if (s.stats_out) {
        double* o = s.stats_out + (size_t)b * RAMP_STEP_STATS_LEN;
#pragma unroll
        for (int k = 0; k < RAMP_STEP_STATS_LEN; ++k) o[k] = st0[k];
    }
    if (s.n_cluster_steps_out) s.n_cluster_steps_out[b] = n_cluster_steps;
}

// RCE:202-295 for every episode; n_jobs_ep (ep.n_jobs_ep, writable) gets every episode's job count
__global__ void ramp_reset_kernel(const EpisodeState ep, int32_t* n_jobs_ep, int32_t n_jobs) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    const int B = ep.B;
    if (b >= B) return;
    n_jobs_ep[b] = n_jobs;
    double* ef = ep.ef; int32_t* ei = ep.ei;
    for (int f = 0; f < EF_COUNT; ++f) EF(f) = 0.0;
    for (int f = 0; f < EI_COUNT; ++f) EI(f) = 0;
    EI(EI_QUEUED) = -1; EI(EI_LAST_SLOT) = -1; EI(EI_PLAN_SLOT) = -1;
    for (int k = 0; k < ep.max_jobs; ++k) {
        ramp_job_record_t& r = ep.rec[(size_t)b * ep.max_jobs + k];
        r.status = RAMP_JS_NOT_ARRIVED; r.event_seq = 0;
        r.time_arrived = r.time_started = r.time_completed = 0.0; r.jct = r.comm = r.comp = r.util = 0.0;
    }
    EF(EF_NEXT_ARRIVAL) = 0.0;                 // RCE:280
    step_get_next_job(ep, hbm_view(ep, b), b); // RCE:281
    EI(EI_QUEUED) = 0;
}

// packs the per-episode scalars for read-back / NCCL all-gather: [B][RAMP_EP_LEN]
__global__ void ramp_export_episode_state_kernel(const EpisodeState ep, double* out) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    const int B = ep.B;
    if (b >= B) return;
    const double* ef = ep.ef; const int32_t* ei = ep.ei;
    double* o = out + (size_t)b * RAMP_EP_LEN;
    o[RAMP_EP_TIME] = EF(EF_NOW); o[RAMP_EP_NEXT_ARRIVAL] = EF(EF_NEXT_ARRIVAL);
    o[RAMP_EP_NUM_ARRIVED] = EI(EI_NUM_ARRIVED); o[RAMP_EP_NUM_COMPLETED] = EI(EI_NUM_COMPLETED);
    o[RAMP_EP_NUM_BLOCKED] = EI(EI_NUM_BLOCKED); o[RAMP_EP_QUEUED_JOB] = EI(EI_QUEUED);
    o[RAMP_EP_NUM_RUNNING] = EI(EI_N_RUNNING); o[RAMP_EP_STEP_COUNTER] = EI(EI_STEP_COUNTER);
    o[RAMP_EP_LOAD_RATE_SUM] = EF(EF_LOAD_SUM); o[RAMP_EP_LOAD_RATE_N] = EI(EI_LOAD_N);
    o[RAMP_EP_DONE] = EI(EI_DONE); o[RAMP_EP_STATUS] = EI(EI_STATUS);
}

// the episode-end finalisation RCE:1123-1167 applied to the EF_ACC_* accumulators: [B][RAMP_ES_LEN].  An episode that is not
// done gets the same formulas over the episode so far.
__global__ void ramp_episode_stats_kernel(const EpisodeState ep, double* out) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    const int B = ep.B;
    if (b >= B) return;
    const double* ef = ep.ef; const int32_t* ei = ep.ei;
    double* o = out + (size_t)b * RAMP_ES_LEN;
    const double t = EF(EF_NOW);                                                  // RCE:1125-1127 (episode_start_time = 0)
    o[RAMP_ES_EPISODE_START_TIME] = 0.0; o[RAMP_ES_EPISODE_END_TIME] = t; o[RAMP_ES_EPISODE_TIME] = t;
    const int n_arr = EI(EI_NUM_ARRIVED), n_comp = EI(EI_NUM_COMPLETED), n_blk = EI(EI_NUM_BLOCKED);
    o[RAMP_ES_NUM_JOBS_ARRIVED] = n_arr; o[RAMP_ES_NUM_JOBS_COMPLETED] = n_comp; o[RAMP_ES_NUM_JOBS_BLOCKED] = n_blk;
    o[RAMP_ES_MEAN_LOAD_RATE] = EI(EI_LOAD_N) > 0 ? __ddiv_rn(EF(EF_LOAD_SUM), (double)EI(EI_LOAD_N)) : 0.0;   // RCE:1129
    o[RAMP_ES_BLOCKING_RATE] = n_arr > 0 ? __ddiv_rn((double)n_blk, (double)n_arr) : 0.0;                       // RCE:1131-1134
    o[RAMP_ES_ACCEPTANCE_RATE] = n_arr > 0 ? __ddiv_rn((double)n_comp, (double)n_arr) : 0.0;                    // RCE:1135-1138
    for (int k = 0; k < 7; ++k) {                                                                                // RCE:1140-1154
        const double info = EF(EF_ACC_INFO + k);
        o[RAMP_ES_COMPUTE_INFO_PROCESSED + k] = info;
        o[RAMP_ES_MEAN_COMPUTE_THROUGHPUT + k] = (info != 0.0 && t != 0.0) ? __ddiv_rn(info, t) : 0.0;
    }
    const double n_steps = EF(EF_ACC_STEPS), n_ticks = EF(EF_ACC_TICKS);                                        // RCE:1156-1167
    const bool live = t != 0.0;
#define RAMP_MEAN(sum, n) ((live && (n) > 0.0) ? __ddiv_rn((sum), (n)) : 0.0)
    o[RAMP_ES_MEAN_COMPUTE_OVERHEAD_FRAC] = RAMP_MEAN(EF(EF_ACC_COMP_FRAC), n_steps);
    o[RAMP_ES_MEAN_COMMUNICATION_OVERHEAD_FRAC] = RAMP_MEAN(EF(EF_ACC_COMM_FRAC), n_steps);
    o[RAMP_ES_MEAN_NUM_JOBS_RUNNING] = RAMP_MEAN(EF(EF_ACC_JOBS_RUNNING), n_steps);
    o[RAMP_ES_MEAN_NUM_MOUNTED_WORKERS] = RAMP_MEAN(EF(EF_ACC_MOUNTED_WORKERS), n_steps);
    o[RAMP_ES_MEAN_MOUNTED_WORKER_UTILISATION_FRAC] = RAMP_MEAN(EF(EF_ACC_UTIL_MOUNTED), n_ticks);
    o[RAMP_ES_MEAN_CLUSTER_WORKER_UTILISATION_FRAC] = RAMP_MEAN(EF(EF_ACC_UTIL_CLUSTER), n_ticks);
#undef RAMP_MEAN
    o[RAMP_ES_NUM_CLUSTER_STEPS] = n_steps; o[RAMP_ES_NUM_TICKS] = n_ticks;
    o[RAMP_ES_DONE] = EI(EI_DONE);
}

#undef EF
#undef EI
#undef VF
#undef VI
#undef VRF
#undef VRI

}  // namespace ramp
