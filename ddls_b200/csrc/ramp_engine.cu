// ramp_engine.cu -- host side of the C ABI declared in include/ramp_b200.h.
//
// Owns the HBM-resident state (templates, memo table, result slots, trace pool, per-episode tables,
// per-CTA scratch slabs) and launches the three kernels of a batched RampClusterEnvironment.step:
//   plan (memo) -> lookahead (persistent CTAs, one lookahead per CTA at a time) -> step (one thread per episode).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <numeric>
#include <utility>
#include <vector>

#include "ramp_kernels.cuh"
#include "ramp_env.cuh"
#include "ramp_env_io.cuh"
#include "ramp_owned.cuh"

using namespace ramp;

namespace {

constexpr int MAX_EVENT_PAIRS = 64;
constexpr int RAMP_SMEM_CARVEOUT = 100;   // percent of the unified L1/shared array given to shared memory

// Templates whose quotient blob does not fit shared memory run on the CTA kernel (one lookahead per CTA).
using LookaheadKernel = void (*)(const LookaheadArgs);
constexpr int32_t RESIDENT_MAX_BYTES = 96 * 1024; // largest quotient blob that goes resident on the thread kernel

LookaheadKernel lookahead_cta_kernel_for(int nt) {   // one CTA of nt threads per lookahead
    switch (nt) {
        case 64: return ramp_lookahead_cta_kernel<2>;
        case 256: return ramp_lookahead_cta_kernel<8>;
        case 128: return ramp_lookahead_cta_kernel<4>;
        default: return nullptr;
    }
}

// the step kernel with 32 episodes per CTA, or 1 when 32 copies of the running-job table do not fit shared memory
using StepKernel = void (*)(const StepArgs);
constexpr size_t STEP_SMEM_MAX = 200 * 1024;
StepKernel step_kernel_for(int nt) { return nt == 32 ? ramp_step_kernel<32> : ramp_step_kernel<1>; }

struct HostTemplate {
    TemplateDev dev;             // copy of what sits in the device array
    DeviceArray<unsigned char> blob;   // single device allocation holding all arrays
    std::vector<unsigned char> bytes;  // canonical host bytes for exact-duplicate detection
    uint64_t hash = 0;
    DeviceArray<unsigned char> res_blob;   // device copy of the quotient blob (thread-per-lookahead kernel), empty if not resident
};

struct ResultArrays {
    DeviceArray<double> jct, comm, comp, util;
    DeviceArray<int32_t> n_ticks, status, util_nmw;
    DeviceArray<int64_t> trace_off;
    cudaError_t alloc(size_t n) { return alloc_each(n, jct, comm, comp, util, n_ticks, status, util_nmw, trace_off); }
    ResultSlots view() const { return {jct.get(), comm.get(), comp.get(), n_ticks.get(), status.get(), trace_off.get(), util.get(), util_nmw.get()}; }
};

struct TraceArrays {
    DeviceArray<int32_t> n_active;
    DeviceArray<double> tick;
    DeviceArray<unsigned long long> top;
    cudaError_t alloc(uint64_t len) {
        const cudaError_t err = alloc_each(len, n_active, tick);
        return err == cudaSuccess ? top.alloc(1) : err;
    }
    TracePool view() const { return TracePool{n_active.get(), tick.get(), top.get(), (uint64_t)n_active.size()}; }
};

// The buffers of one step's lookaheads when steps overlap (ramp_step_device): the speculative plan and bucket run on the plan
// stream, the thread kernel on the window's stream, and the commit, the repair launch and the step kernel on the engine stream.
// ev_consumed marks the end of the repair launch that used the window last, the last reader of its lists; the window's next
// plan waits for it.  A window holds only its lists (about 0.56 KB per episode); the thread kernel's HBM slabs are one pool
// shared by every launch.  N_WINDOWS (DESIGN.md §4): enough windows that planning a step never waits for a window while the
// SMs have free thread-kernel slots.
constexpr int N_WINDOWS = 16;
struct LookaheadWindow {
    Stream stream;
    Event ev_planned, ev_end, ev_consumed;
    DeviceArray<Counters> counters;
    DeviceArray<WorkItem> items_res, chunk_items;   // [B], [B][32]
    DeviceArray<ChunkDesc> chunks;                  // [B]
    DeviceArray<int32_t> rank, tcount, tbase;       // [B], [max_templates + 1] x 2
    DeviceArray<SpecRecord> rec;                    // [B]
};

}  // namespace

struct ramp_engine {
    ramp_config_t cfg{};
    int sm_count = 0;
    Stream stream;
    // templates
    std::vector<HostTemplate> templates;
    DeviceArray<TemplateDev> d_templates;
    uint64_t max_scratch = 0;
    int32_t max_w = 1, max_c = 1;
    int32_t par_cap = 0;         // bytes of shared-memory parent counters per lookahead
    // memo + results
    uint32_t memo_cap = 0;
    DeviceArray<unsigned long long> d_memo_keys;
    DeviceArray<int32_t> d_memo_vals;
    DeviceArray<unsigned long long> d_memo_keys2;
    uint32_t memo_cap2 = 0;
    ResultArrays res;
    int32_t n_slots = 0;
    TraceArrays pool;
    // per-step
    DeviceArray<WorkItem> d_items;
    DeviceArray<Counters> d_counters;
    DeviceArray<MemoStats> d_stats;      // [0] the cumulative counters the kernels add to, [1] their copy at the last ramp_reset
    DeviceArray<ramp_action_t> d_actions;
    DeviceArray<double> d_step_stats;
    DeviceArray<int32_t> d_n_cluster_steps;
    DeviceArray<double> d_ep_export;
    DeviceArray<double> d_es_export;     // [B][RAMP_ES_LEN] ramp_get_episode_stats
    // episode state: the view the kernels take, and its arrays
    EpisodeState ep{};
    DeviceArray<double> ep_ef, ep_es, ep_rf, tick_util; DeviceArray<int32_t> ep_ei, ep_ri, tick_util_n; DeviceArray<ramp_job_record_t> ep_rec;
    DeviceArray<ramp_arrival_t> d_arrivals;
    DeviceArray<int32_t> d_n_jobs_ep;
    // ramp_reset copies the caller's arrivals here and uploads them from here, so it returns without waiting for the upload;
    // ev_stage marks the end of the last upload, which the next reset waits for before it writes the buffer again
    PinnedArray<ramp_arrival_t> h_arr_stage;
    Event ev_stage;
    // ramp_step_kernel: threads per CTA (one per episode) and its dynamic shared memory (the episodes' state on chip)
    int step_nt = 0;
    size_t step_smem = 0;
    // lookahead scratch
    DeviceArray<unsigned char> d_scratch;
    uint64_t scratch_stride = 0;
    // CTA-per-lookahead kernel (templates that are not resident)
    int cta_nt = 0;              // 0 = pick 256, 128 or 64 threads per launch; RAMP_LOOKAHEAD_CTA_THREADS forces one
    int cta_grid = 0;            // resident CTAs of the 128-thread variant
    int cta64_grid = 0;          // resident CTAs of the 64-thread variant
    int cta256_grid = 0;         // resident CTAs of the 256-thread variant
    int cta_grid_for(int nt) const { return nt == 256 ? cta256_grid : nt == 128 ? cta_grid : cta64_grid; }
    size_t cta_smem_bytes = 0;
    int debug = 0;               // RAMP_DEBUG=1 prints the launch decisions to stderr
    bool cta_only = false;       // RAMP_LOOKAHEAD_MODE=cta: nothing resident, every lookahead on the CTA kernel
    PinnedArray<int32_t> h_n_work;   // [1] read-back of Counters::n_work
    PinnedArray<MemoStats> h_stats;  // [2] read-back of d_stats
    // resident (quotient) templates: thread-per-lookahead kernel
    int use_quotient = 1;        // 0 (RAMP_LOOKAHEAD_MODE=thread_unfolded): resident blobs are built from the unfolded job (identity quotient)
    int n_resident = 0, n_nonresident = 0;
    int32_t res_tmpl_cap = 0, res_n_cap = 0, res_spill_ops = 0, res_spill_deps = 0;
    int res_grid = 0;
    int res_per_sm = 0;                    // thread-kernel CTAs one SM holds at once
    size_t res_smem = 0;
    DeviceArray<unsigned char> d_res_scratch;   // the slab pool: [sm_count][res_per_sm][res_scratch_stride], shared by every launch
    DeviceArray<uint32_t> d_res_slab_mask;      // [sm_count]: the slabs held by running CTAs (ramp_lookahead_thread.cuh)
    uint64_t res_scratch_stride = 0;
    DeviceArray<WorkItem> d_items_res;
    DeviceArray<WorkItem> d_chunk_items;   // [B][32]
    DeviceArray<ChunkDesc> d_chunks;       // [B]
    DeviceArray<int32_t> d_tcount;         // [max_templates + 1]
    DeviceArray<int32_t> d_tbase;
    DeviceArray<int32_t> d_rank;           // [B]
    DeviceArray<TemplateHints> d_hints;    // [max_templates]
    DeviceArray<double> d_hint_jct;        // [max_templates]
    // device-resident rollouts (ramp_env_*)
    bool has_env = false;
    EnvDev env{};
    std::vector<DeviceArray<unsigned char>> env_allocs;
    PinnedArray<int32_t> env_h_need;     // [0] = count, [1] = error flag; [2], [3]: the same, read by ramp_env_read; [4] engine error episode
                                         // [6..7] ramp_env_ingest's range word
    PinnedArray<unsigned char> env_h_mirror;   // host arrays of ramp_env_host_mirror
    bool env_unchecked_decide = false;   // a ramp_env_decide without need_host_out has not been looked at yet
    bool env_agents_set = false;         // ramp_env_set_agents ran
    // device placement of uneven jobs (ramp_env_set_placer_tables); the geometry table's host copy decides every insertion
    bool has_placer = false;
    int32_t env_shape[3] = {0, 0, 0};
    PlaceDev place{};
    std::vector<unsigned long long> place_keys;         // [cap][n_words + 1], as the device table
    std::vector<int32_t> place_tids;                    // [cap]
    uint32_t place_count = 0;
    DeviceArray<unsigned long long> place_table_keys;
    DeviceArray<int32_t> place_table_tid;
    DeviceArray<double> steplog_stats, steplog_rewards;   // ramp_env_steplog_begin: [horizon][RAMP_ENV_STEP_STATS_LEN][B], [horizon][B]
    DeviceArray<int32_t> steplog_actions;                 // [horizon][B]
    // i/o in caller-owned device memory (ramp_env_ingest / ramp_env_export), allocated by the first call that needs them
    DeviceArray<float> env_graph_static;                  // [n_models][6] ramp_env_set_graph_static
    DeviceArray<unsigned long long> env_range_err;        // [1] ramp_env_ingest_kernel's sticky word
    DeviceArray<long long> env_range_val;                 // [B] the out-of-set action recorded with it
    Event env_ev_to_caller, env_ev_to_engine;             // the caller's stream waits for the engine's / the engine's for the caller's
    DeviceArray<uint32_t> env_ingest_seq;                 // [2] ramp_env_ingest_kernel's call number and CTA count (EnvIngestArgs)
    bool env_range_armed = false;                         // a ramp_env_ingest ran since the word was last looked at
    // CUDA-graph capture of the torch steps (ramp_env_ingest on a capturing stream, DESIGN.md §7 g)
    bool env_captured = false;           // a whole step was captured: its replays leave their errors unannounced to the host
    int64_t sized_templates = -1;        // the template count the last eager ramp_step_device sized the scratch for (-1: none)
    // standalone lookahead buffers
    DeviceArray<WorkItem> sa_chunk_items;
    DeviceArray<ChunkDesc> sa_chunks;
    ResultArrays sa_res;
    int32_t sa_cap = 0;
    DeviceArray<WorkItem> sa_items;      // [n]: the non-resident and resident work lists, one after the other
    DeviceArray<int32_t> sa_rank;        // [n] ramp_bucket_kernel scratch
    DeviceArray<Counters> sa_counters;
    // overlapped steps (ramp_step_device, DESIGN.md §4)
    int overlap = 1;                     // RAMP_STEP_OVERLAP=0: every step takes the in-order path
    LookaheadWindow win[N_WINDOWS];      // allocated by the first overlapped step
    bool win_ready = false;
    uint64_t win_seq = 0;
    Stream plan_stream;
    Event ev_reset;                      // the last ramp_reset's table clears; the next speculative plan waits for it
    bool reset_pending = false;
    DeviceArray<unsigned long long> d_spec_keys, d_repair_keys;   // [memo_cap] each: the result and repair tables
    int32_t spec_base = 0, repair_base = 0;                         // their result slots: [spec_base, spec_base + 2 memo_cap)
    // instrumentation
    int64_t launches = 0;
    Event ev_a[MAX_EVENT_PAIRS], ev_b[MAX_EVENT_PAIRS];
    int ev_pending = 0;
    double la_ms_union = 0.0;            // union of the event pairs' intervals (overlapped windows count once)
    double la_ms_total = 0.0;
    int64_t la_launches = 0;
    unsigned long long la_items_base = 0, la_bytes_base = 0, la_qbytes_base = 0;
};

// A kernel's dynamic shared memory limit (cudaFuncAttributeMaxDynamicSharedMemorySize) belongs to the kernel in the device's
// context, not to an engine: every engine of the process shares it.  Lowering it to what one engine needs would make another
// engine's launches that need more fail, so it only ever rises.  Each engine still launches with, and sizes its grid for, its own
// dynamic shared memory.
cudaError_t ramp::reserve_dynamic_smem(const void* kern, size_t bytes) {
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, size_t> reserved;
    int dev = 0;
    cudaError_t err = cudaGetDevice(&dev);
    if (err != cudaSuccess) return err;
    std::lock_guard<std::mutex> lock(mu);
    size_t& cur = reserved[{dev, kern}];
    if (bytes <= cur) return cudaSuccess;
    err = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (err == cudaSuccess) cur = bytes;
    return err;
}

namespace {

// adds the pending event pairs to the lookahead time: their sum, and the union of their intervals (the pairs of overlapped
// steps' windows run at the same time, so only the union is a share of the steps' time)
int resolve_events(ramp_engine* e) {
    std::vector<std::pair<float, float>> iv;
    for (int k = 0; k < e->ev_pending; ++k) {
        float ms = 0.f, t0 = 0.f;
        CUDA_TRY(cudaEventElapsedTime(&ms, e->ev_a[k].get(), e->ev_b[k].get()));
        CUDA_TRY(cudaEventElapsedTime(&t0, e->ev_a[0].get(), e->ev_a[k].get()));
        e->la_ms_total += ms;
        e->la_launches++;
        iv.emplace_back(t0, t0 + ms);
    }
    std::sort(iv.begin(), iv.end());
    for (size_t k = 0; k < iv.size();) {
        float lo = iv[k].first, hi = iv[k].second;
        for (++k; k < iv.size() && iv[k].first <= hi; ++k) hi = std::max(hi, iv[k].second);
        e->la_ms_union += hi - lo;
    }
    e->ev_pending = 0;
    return RAMP_OK;
}

// (re)allocates the per-CTA scratch slabs for the largest registered template and picks the CTA kernel's grids
int ensure_scratch(ramp_engine* e) {
    const uint64_t trace_bytes = align_up((uint64_t)e->cfg.trace_cap * 12, 16);
    const uint64_t stride = align_up(std::max<uint64_t>(e->max_scratch, 16), 256) + align_up(trace_bytes, 256);
    const size_t cta_smem = lookahead_cta_smem(e->max_w, e->max_c, e->par_cap);
    if (cta_smem > 200 * 1024)
        return set_error(RAMP_ERR_CAPACITY, "a template needs %zu B of shared memory (max 200 KiB)", cta_smem);
    if (cta_smem != e->cta_smem_bytes || e->cta_grid == 0) {
        for (int nt : {256, 128, 64}) {
            LookaheadKernel kern = lookahead_cta_kernel_for(nt);
            CUDA_TRY(reserve_dynamic_smem((const void*)kern, cta_smem));
            CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, RAMP_SMEM_CARVEOUT));
            int occ = 0;
            CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, nt, cta_smem));
            if (occ < 1) occ = 1;
            // persistent CTAs: a whole number of waves (SMs x resident CTAs per SM)
            (nt == 256 ? e->cta256_grid : nt == 128 ? e->cta_grid : e->cta64_grid) = e->sm_count * occ;
        }
        e->cta_smem_bytes = cta_smem;
    }
    // one slab per CTA of the largest grid: one CTA kernel runs at a time, on the engine stream
    const int n_slabs = std::max({e->cta256_grid, e->cta_grid, e->cta64_grid});
    if (stride != e->scratch_stride || stride * (uint64_t)n_slabs != e->d_scratch.size()) {
        CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
        CUDA_TRY(e->d_scratch.alloc(stride * (uint64_t)n_slabs));
        e->scratch_stride = stride;
    }
    return RAMP_OK;
}

LookaheadArgs make_lookahead_args(ramp_engine* e, const WorkItem* items, Counters* counters, const ResultSlots& res,
                                  const TracePool& pool, MemoStats* stats) {
    LookaheadArgs a{};
    a.templates = e->d_templates.get();
    a.items = items;
    a.n_work = &counters->n_work;
    a.cursor = &counters->work_cursor;
    a.scratch = e->d_scratch.get();
    a.scratch_stride = e->scratch_stride;
    a.res = res;
    a.pool = pool;
    a.trace_cap = e->cfg.trace_cap;
    a.w_cap = e->max_w;
    a.c_cap = e->max_c;
    a.par_cap = e->par_cap;
    a.stats = stats;
    return a;
}

uint64_t fnv1a(const unsigned char* p, size_t n) {
    uint64_t h = 1469598103934665603ull;
    for (size_t i = 0; i < n; ++i) { h ^= p[i]; h *= 1099511628211ull; }
    return h;
}

// rank keys: larger key wins.  Sorting by (priority desc, index asc) and numbering from the top reproduces
// "iterate in sorted() order, replace only on strictly greater priority" (RCE:56-66, RCE:672-685).
void make_rank_keys(const int64_t* prio, int32_t n, std::vector<uint32_t>& key) {
    std::vector<int32_t> order(n);
    std::iota(order.begin(), order.end(), 0);
    std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return prio[a] > prio[b]; });
    key.resize(n);
    for (int32_t r = 0; r < n; ++r) key[order[r]] = (uint32_t)(n - r);
}


// ---- resident (quotient) templates ---------------------------------------------------------------------------
int bits_for_u64(uint64_t max_value) { int b = 1; while ((max_value >> b) != 0) ++b; return b; }

// Packs a quotient job (ramp_quotient.cpp) into the blob the thread-per-lookahead kernel bulk-copies into shared memory
// (layout: ResHeader, ramp_lookahead_thread.cuh).  Returns false when the job is not eligible: blob larger than
// max_bytes, more channel groups than the kernel's winner table holds (RAMP_T_CCAP), class sizes / counters beyond 16
// bits, or a dep word wider than 64 bits.
bool build_resident_blob(const ramp_lowered_job_t* j, const ramp_quotient_t& q, int32_t max_bytes, std::vector<unsigned char>& blob) {
    const int32_t N = q.n_ops, E = q.n_deps;
    if (N < 1 || q.n_workers > 0xFFFF || q.n_channels > RAMP_T_CCAP) return false;
    if (!q.masks_valid) return false;
    std::vector<uint64_t> in_total(N, 0);
    uint32_t max_inc = 1;
    // keys only order entries: re-rank them densely so that the key and the group set share one 32-bit word
    std::vector<uint32_t> distinct(q.dep_key, q.dep_key + E);
    std::sort(distinct.begin(), distinct.end());
    distinct.erase(std::unique(distinct.begin(), distinct.end()), distinct.end());
    std::vector<uint32_t> dense_key(E);
    for (int32_t k = 0; k < E; ++k) {
        in_total[q.dep_dst[k]] += q.dep_inc[k];
        max_inc = std::max(max_inc, q.dep_inc[k]);
        dense_key[k] = (uint32_t)(std::lower_bound(distinct.begin(), distinct.end(), q.dep_key[k]) - distinct.begin()) + 1u;
    }
    for (int32_t c = 0; c < N; ++c)
        if (q.op_weight[c] > 0xFFFF || in_total[c] > 0xFFFF || q.op_threshold[c] > 0xFFFFFFFFu) return false;   // u16 counters never wrap
    const int kbits = bits_for_u64((uint64_t)distinct.size() + 1), cbits = std::max(q.n_channels, 1);
    const int ibits = bits_for_u64(max_inc), nbits = bits_for_u64((uint64_t)N);
    if (kbits + cbits > 32 || 1 + ibits + nbits > 32) return false;     // dep word = two 32-bit halves: key | group set, flow | inc | child
    std::vector<int32_t> in_deg(N, 0), src;
    for (int32_t k = 0; k < E; ++k) in_deg[q.dep_dst[k]]++;
    for (int32_t c = 0; c < N; ++c) if (in_deg[c] == 0) src.push_back(c);
    ResHeader h{};
    h.n_ops = N; h.n_deps = E; h.n_workers = q.n_workers; h.n_channels = q.n_channels;
    h.n_src = (int32_t)src.size(); h.num_training_steps = j->num_training_steps; h.orig_workers = j->n_workers;
    h.kmask = (uint32_t)((1ull << kbits) - 1ull); h.cmask = (uint32_t)((1ull << cbits) - 1ull); h.imask = (uint32_t)((1ull << ibits) - 1ull);
    h.cshift = kbits; h.fshift = 0; h.ishift = 1; h.dshift = 1 + ibits;
    size_t off = sizeof(ResHeader);
    const size_t off_rec = off;                 off += align_up((uint64_t)N * 16, 16);
    h.off_op_row = (int32_t)off;                off += align_up((uint64_t)N * 8, 16);
    h.off_op_thr = (int32_t)off;                off += align_up((uint64_t)N * 4, 16);
    h.off_out = (int32_t)off;                   off += align_up((uint64_t)std::max(E, 1) * 16, 16);
    h.off_src = (int32_t)off;                   off += align_up((uint64_t)std::max<size_t>(src.size(), 1) * 4, 16);
    if (off > (size_t)max_bytes) return false;
    h.total_bytes = (int32_t)off;
    blob.assign(off, 0);
    memcpy(blob.data(), &h, sizeof(h));
    struct OpRec { double cost; uint32_t key; uint32_t worker; };
    OpRec* rec = reinterpret_cast<OpRec*>(blob.data() + off_rec);
    int32_t* row = reinterpret_cast<int32_t*>(blob.data() + h.off_op_row);
    uint32_t* thr = reinterpret_cast<uint32_t*>(blob.data() + h.off_op_thr);
    struct OutRec { double run_time; uint32_t lo, hi; };      // = the ready-flow frontier entry the kernel copies it to
    static_assert(sizeof(OutRec) == 16, "out-entry record is 16 bytes");
    OutRec* out = reinterpret_cast<OutRec*>(blob.data() + h.off_out);
    for (int32_t c = 0; c < N; ++c) {
        rec[c] = OpRec{q.op_cost[c] + 0.0, q.op_key[c], q.op_worker[c] | (q.op_weight[c] << 16)};
        thr[c] = q.op_threshold[c];
        // the class's out-entries, flows first, in descending key order (the order the kernel keeps its ready-flow frontier
        // in: completing the class merges them into it), then the non-flows in entry order
        std::vector<int32_t> ent;
        for (int32_t k = q.row_ptr[c]; k < q.row_ptr[c + 1]; ++k) if (q.dep_is_flow[k] != 0) ent.push_back(k);
        std::stable_sort(ent.begin(), ent.end(), [&](int32_t a, int32_t b) { return dense_key[a] > dense_key[b]; });
        const int32_t n_fl = (int32_t)ent.size();
        for (int32_t k = q.row_ptr[c]; k < q.row_ptr[c + 1]; ++k) if (q.dep_is_flow[k] == 0) ent.push_back(k);
        int32_t pos = q.row_ptr[c];
        for (const int32_t k : ent) {
            const uint32_t lo = dense_key[k] | (uint32_t)(q.dep_group_mask[k] << h.cshift);
            const uint32_t hi = (q.dep_is_flow[k] ? 1u : 0u) | (q.dep_inc[k] << h.ishift) | ((uint32_t)q.dep_dst[k] << h.dshift);
            out[pos++] = OutRec{q.dep_run_time[k] + 0.0, lo, hi};
        }
        const int32_t n_nf = q.row_ptr[c + 1] - q.row_ptr[c] - n_fl;
        if (n_fl > 0xFFFF || n_nf > 0x7FFF) return false;
        row[2 * c] = q.row_ptr[c]; row[2 * c + 1] = n_fl | (n_nf << 16);
    }
    if (!src.empty()) memcpy(blob.data() + h.off_src, src.data(), sizeof(int32_t) * src.size());
    return true;
}

// the identity quotient: every op its own class (RAMP_LOOKAHEAD_MODE=thread_unfolded; lets the tests run the thread kernel
// on unfolded jobs)
int identity_quotient(const ramp_lowered_job_t* j, ramp_quotient_t* q) {
    memset(q, 0, sizeof(*q));
    const int32_t N = j->n_ops, E = j->n_deps;
    std::vector<uint32_t> ok, dk;
    make_rank_keys(j->op_prio, N, ok);
    make_rank_keys(j->dep_prio, E, dk);
    q->n_ops = N; q->n_deps = E; q->n_workers = j->n_workers; q->n_channels = j->n_channels;
    q->op_cost = (double*)malloc(sizeof(double) * N); q->op_key = (uint32_t*)malloc(4 * (size_t)N); q->op_worker = (uint32_t*)malloc(4 * (size_t)N);
    q->op_weight = (uint32_t*)malloc(4 * (size_t)N); q->op_threshold = (uint32_t*)malloc(4 * (size_t)N); q->row_ptr = (int32_t*)malloc(4 * ((size_t)N + 1));
    const size_t e1 = std::max(E, 1);
    q->dep_dst = (int32_t*)malloc(4 * e1); q->dep_run_time = (double*)malloc(8 * e1); q->dep_key = (uint32_t*)malloc(4 * e1);
    q->dep_channel = (uint32_t*)malloc(4 * e1); q->dep_is_flow = (uint8_t*)malloc(e1); q->dep_inc = (uint32_t*)malloc(4 * e1);
    q->dep_group_mask = (uint64_t*)malloc(8 * e1); q->merged = 0; q->masks_valid = j->n_channels <= 64 ? 1 : 0;
    q->op_class = (int32_t*)malloc(4 * (size_t)N); q->dep_entry = (int32_t*)malloc(4 * e1);
    for (int32_t i = 0; i < N; ++i) {
        q->op_cost[i] = j->op_cost[i]; q->op_key[i] = ok[i]; q->op_worker[i] = j->op_worker[i]; q->op_weight[i] = 1;
        q->op_threshold[i] = j->op_n_parents[i]; q->row_ptr[i] = j->row_ptr[i]; q->op_class[i] = i;
    }
    q->row_ptr[N] = j->row_ptr[N];
    for (int32_t k = 0; k < E; ++k) {
        q->dep_dst[k] = j->dep_dst[k]; q->dep_run_time[k] = j->dep_run_time[k]; q->dep_key[k] = dk[k];
        q->dep_channel[k] = (j->dep_channel[k] == RAMP_NO_CHANNEL) ? 0xFFFFFFFFu : (uint32_t)j->dep_channel[k];
        q->dep_group_mask[k] = (j->dep_channel[k] == RAMP_NO_CHANNEL || !q->masks_valid) ? 0ull : (1ull << j->dep_channel[k]);
        q->dep_is_flow[k] = j->dep_is_flow[k] ? 1 : 0; q->dep_inc[k] = 1; q->dep_entry[k] = k;
    }
    return RAMP_OK;
}

// shared memory / grid / HBM slabs of the thread-per-lookahead kernel for the resident templates registered so far
int ensure_thread_scratch(ramp_engine* e) {
    const size_t need = thread_smem_bytes(e->res_tmpl_cap, e->res_n_cap);
    if (need > 220 * 1024) return set_error(RAMP_ERR_CAPACITY, "resident templates need %zu B of shared memory (max 220 KiB)", need);
    // At most 2 CTAs per SM, whichever launches they belong to: a CTA asks for at least the shared memory that keeps a third
    // one off the SM.  Two CTAs are four warps, one per scheduler of the SM; with a third, two sim warps share a scheduler,
    // and on config 3 the overlapped step got slower (DESIGN.md §4).
    int sm_smem = 0, blk_reserved = 0;
    CUDA_TRY(cudaDeviceGetAttribute(&sm_smem, cudaDevAttrMaxSharedMemoryPerMultiprocessor, e->cfg.device));
    CUDA_TRY(cudaDeviceGetAttribute(&blk_reserved, cudaDevAttrReservedSharedMemoryPerBlock, e->cfg.device));
    cudaFuncAttributes fa{};
    CUDA_TRY(cudaFuncGetAttributes(&fa, ramp_lookahead_thread_kernel));
    const size_t three = (size_t)sm_smem / 3 - fa.sharedSizeBytes - (size_t)blk_reserved;   // the most at which 3 CTAs fit
    const size_t smem = std::max(need, align_up((uint64_t)three + 1, 128));
    if (smem != e->res_smem || e->res_grid == 0) {
        CUDA_TRY(reserve_dynamic_smem((const void*)ramp_lookahead_thread_kernel, smem));
        CUDA_TRY(cudaFuncSetAttribute(ramp_lookahead_thread_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, RAMP_SMEM_CARVEOUT));
        int occ = 0;
        CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, ramp_lookahead_thread_kernel, RAMP_THREAD_CTA, smem));
        occ = std::max(occ, 1);
        // one chunk = up to 32 lookaheads; enough resident CTAs for every episode to miss at once
        const int want = (e->cfg.n_episodes + 31) / 32 + 8;
        e->res_grid = std::max(1, std::min(e->sm_count * occ, want));
        e->res_per_sm = occ;
        e->res_smem = smem;
        if (e->debug) fprintf(stderr, "[ramp] thread kernel: %zu B dynamic shared memory (%zu B needed), %d CTAs of %d threads per SM fit, grid %d\n",
                              smem, need, occ, RAMP_THREAD_CTA, e->res_grid);
    }
    // one slab per CTA that can be resident, whichever launch it belongs to: every thread kernel in flight is ordered before
    // the engine stream's end (a window's kernel before its step's commit)
    const uint64_t stride = thread_scratch_bytes(e->res_spill_ops, e->res_spill_deps, e->cfg.trace_cap);
    const uint64_t n_slabs = (uint64_t)e->sm_count * (uint64_t)e->res_per_sm;
    if (stride != e->res_scratch_stride || stride * n_slabs != e->d_res_scratch.size()) {
        CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
        CUDA_TRY(e->d_res_scratch.alloc(stride * n_slabs));
        if (e->d_res_slab_mask.size() != (size_t)e->sm_count) CUDA_TRY(e->d_res_slab_mask.alloc((size_t)e->sm_count));
        CUDA_TRY(cudaMemset(e->d_res_slab_mask.get(), 0, sizeof(uint32_t) * (size_t)e->sm_count));
        e->res_scratch_stride = stride;
    }
    return RAMP_OK;
}

ThreadArgs make_thread_args(ramp_engine* e, const ChunkDesc* chunks, const WorkItem* chunk_items, Counters* c,
                            const ResultSlots& res, const TracePool& pool, MemoStats* stats) {
    ThreadArgs a{};
    a.templates = e->d_templates.get(); a.chunks = chunks; a.n_chunks = &c->n_chunks; a.cursor = &c->chunk_cursor; a.items = chunk_items;
    a.scratch = e->d_res_scratch.get(); a.scratch_stride = e->res_scratch_stride;
    a.slab_mask = e->d_res_slab_mask.get(); a.slab_groups = e->sm_count; a.slabs_per_sm = e->res_per_sm;
    a.res = res; a.pool = pool; a.trace_cap = e->cfg.trace_cap;
    a.tmpl_cap = e->res_tmpl_cap; a.n_cap = e->res_n_cap; a.spill_ops = e->res_spill_ops; a.spill_deps = e->res_spill_deps;
    a.stats = stats; a.hints = e->d_hints.get(); a.hint_jct = e->d_hint_jct.get();
    return a;
}

// groups the resident work items (list 2 of `c`) by template into chunks of <= 32 for the thread kernel, on the device
void bucket_resident(ramp_engine* e, const WorkItem* items, Counters* c, WorkItem* chunk_items, ChunkDesc* chunks, int32_t* rank,
                     int32_t* tcount, int32_t* tbase, cudaStream_t st) {
    BucketArgs ba{};
    ba.items = items; ba.n_items = &c->n_work_res; ba.n_templates = (int32_t)e->templates.size();
    ba.tcount = tcount; ba.tbase = tbase; ba.chunk_items = chunk_items; ba.chunks = chunks;
    ba.n_chunks = &c->n_chunks; ba.cursor = &c->chunk_cursor; ba.rank = rank;
    ramp_bucket_kernel<<<1, 1024, 0, st>>>(ba);
    e->launches++;
}

// Launches the lookaheads of a step or of a standalone run (ramp_run_lookaheads), so both pick kernels by the same rule.
// The resident ones, already bucketed into chunks, run on the thread kernel over thread_grid CTAs (0: there are none).  The
// n others (list 0 of `c`, a count the host knows) run on the CTA kernel after them.
int launch_lookaheads(ramp_engine* e, const ChunkDesc* chunks, const WorkItem* chunk_items, int thread_grid,
                      const WorkItem* items, int n, Counters* c, const ResultSlots& res, const TracePool& pool,
                      MemoStats* stats, cudaStream_t st) {
    if (thread_grid > 0) {
        ThreadArgs ta = make_thread_args(e, chunks, chunk_items, c, res, pool, stats);
        ramp_lookahead_thread_kernel<<<thread_grid, RAMP_THREAD_CTA, e->res_smem, st>>>(ta);
        e->launches++;
    }
    if (n == 0) return RAMP_OK;
    // Each lookahead sets the latency.  While they all fit the SMs at once (registers cap the CTA kernel at cta_grid x 4
    // warps) each gets a 256-thread CTA if 8 warps per lookahead still fit (2.4 ms instead of 2.9 ms for the bench job), else a
    // 128-thread CTA; beyond that 64-thread CTAs, persistent over as many waves as it takes.  RAMP_LOOKAHEAD_CTA_THREADS
    // overrides the thread count.
    const int reg_slots = e->cta_grid * 4;
    int nt = 64;
    if (n <= e->cta256_grid && 8 * n <= reg_slots) nt = 256;
    else if (n <= e->cta_grid && 4 * n <= reg_slots) nt = 128;
    if (e->cta_nt) nt = e->cta_nt;
    const int grid = std::min(n, e->cta_grid_for(nt));
    if (e->debug) fprintf(stderr, "[ramp] lookaheads: non-resident=%d reg_slots=%d -> CTA threads %d, grid %d\n", n, reg_slots, nt, grid);
    lookahead_cta_kernel_for(nt)<<<grid, nt, e->cta_smem_bytes, st>>>(make_lookahead_args(e, items, c, res, pool, stats));
    e->launches++;
    return RAMP_OK;
}

// one array of the device environment (EnvDev), owned by the engine: n elements of T from `src`, or zeros
template <class T> int env_upload(ramp_engine* e, T** dst, const void* src, size_t n) {
    e->env_allocs.emplace_back();
    CUDA_TRY(e->env_allocs.back().alloc(sizeof(T) * std::max<size_t>(n, 1)));
    *dst = reinterpret_cast<T*>(e->env_allocs.back().get());
    if (src && n) CUDA_TRY(cudaMemcpy(e->env_allocs.back().get(), src, sizeof(T) * n, cudaMemcpyHostToDevice));
    else CUDA_TRY(cudaMemset(e->env_allocs.back().get(), 0, sizeof(T) * std::max<size_t>(n, 1)));
    return RAMP_OK;
}

// makes `to` wait for the work queued on `from` so far
int env_fence(cudaEvent_t ev, cudaStream_t from, cudaStream_t to) {
    CUDA_TRY(cudaEventRecord(ev, from));
    CUDA_TRY(cudaStreamWaitEvent(to, ev, 0));
    return RAMP_OK;
}

// A step captured into a CUDA graph must need nothing from the host: a replay runs no host code, so the launch shapes and buffers
// the step uses must already be fixed by eager steps (DESIGN.md §7 g).  Checked before a captured step enqueues anything.
int capture_refusal(ramp_engine* e) {
    if (e->n_nonresident > 0)
        return set_error(RAMP_ERR_BAD_ARG, "CUDA-graph capture refused: %d template(s) run on the CTA kernel, whose launch shape needs "
                         "the step's work count on the host", e->n_nonresident);
    if (e->sized_templates < 0)
        return set_error(RAMP_ERR_BAD_ARG, "CUDA-graph capture refused: no eager step has run yet to size the engine's buffers");
    if (e->sized_templates != (int64_t)e->templates.size())
        return set_error(RAMP_ERR_BAD_ARG, "CUDA-graph capture refused: %lld template(s) were registered since the last eager step, "
                         "so the lookahead scratch may have to grow", (long long)e->templates.size() - (long long)e->sized_templates);
    return RAMP_OK;
}

// the range word and the events of ramp_env_ingest / ramp_env_export, made by the first of them; the word is cleared on the
// engine stream, which both calls fence their kernels behind
int env_io_ready(ramp_engine* e) {
    if (e->env_ev_to_engine) return RAMP_OK;
    CUDA_TRY(e->env_range_err.alloc(1));
    CUDA_TRY(e->env_range_val.alloc((size_t)e->env.B));
    CUDA_TRY(e->env_ingest_seq.alloc(2));
    CUDA_TRY(cudaMemsetAsync(e->env_range_err.get(), 0xFF, sizeof(unsigned long long), e->stream.get()));
    CUDA_TRY(cudaMemsetAsync(e->env_ingest_seq.get(), 0, 2 * sizeof(uint32_t), e->stream.get()));
    CUDA_TRY(create(e->env_ev_to_caller, cudaEventDisableTiming));
    CUDA_TRY(create(e->env_ev_to_engine, cudaEventDisableTiming));
    return RAMP_OK;
}

// queues the copy of the range word to env_h_need[6..7]; the caller synchronises the engine stream before env_range_raise
int env_range_fetch(ramp_engine* e) {
    CUDA_TRY(cudaMemcpyAsync(e->env_h_need.get() + 6, e->env_range_err.get(), sizeof(unsigned long long), cudaMemcpyDeviceToHost,
                             e->stream.get()));
    return RAMP_OK;
}

// RJPE:314-316 for the first out-of-set action ramp_env_ingest recorded, if any.  Raising clears the word and the step's invalid-
// action word, as the step that raised is not taken any further.
int env_range_raise(ramp_engine* e) {
    e->env_range_armed = false;
    const unsigned long long w = *reinterpret_cast<const unsigned long long*>(e->env_h_need.get() + 6);
    if (w == ENV_NO_RANGE_ERR) return RAMP_OK;
    const int b = (int)(uint32_t)w;
    long long a = 0;
    CUDA_TRY(cudaMemcpy(&a, e->env_range_val.get() + b, sizeof(long long), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemsetAsync(e->env_range_err.get(), 0xFF, sizeof(unsigned long long), e->stream.get()));
    CUDA_TRY(cudaMemsetAsync(e->env.err, 0, sizeof(int32_t), e->stream.get()));
    CUDA_TRY(cudaMemsetAsync(e->env_ingest_seq.get(), 0, sizeof(uint32_t), e->stream.get()));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    std::string set;
    for (int k = 0; k <= e->env.max_degree; ++k) set += (k ? ", " : "") + std::to_string(k);
    return set_error(RAMP_ERR_BAD_ARG, "episode %d: Action %lld not in action set [%s]. (RJPE:314-316)", b, a, set.c_str());
}

// the action rows the engine writes itself, in stream order (ramp_step_host, the device environment): their steps take the
// in-order path
bool engine_owned(const ramp_engine* e, const void* p) {
    const uintptr_t q = (uintptr_t)p;
    auto in = [q](const void* base, size_t bytes) { return q >= (uintptr_t)base && q < (uintptr_t)base + bytes; };
    if (in(e->d_actions.get(), sizeof(ramp_action_t) * e->d_actions.size())) return true;
    for (const auto& a : e->env_allocs) if (in(a.get(), a.size())) return true;
    return false;
}

// the windows' buffers
int ensure_windows(ramp_engine* e) {
    const int B = e->cfg.n_episodes;
    const size_t nt = (size_t)e->cfg.max_templates + 1;
    if (!e->win_ready) {
        CUDA_TRY(create(e->plan_stream, cudaStreamNonBlocking));
        CUDA_TRY(create(e->ev_reset, cudaEventDisableTiming));
        for (LookaheadWindow& w : e->win) {
            CUDA_TRY(create(w.stream, cudaStreamNonBlocking));
            CUDA_TRY(create(w.ev_planned, cudaEventDisableTiming));
            CUDA_TRY(create(w.ev_end, cudaEventDisableTiming));
            CUDA_TRY(create(w.ev_consumed, cudaEventDisableTiming));
            CUDA_TRY(w.counters.alloc(1));
            CUDA_TRY(cudaMemset(w.counters.get(), 0, sizeof(Counters)));
            CUDA_TRY(alloc_each(B, w.items_res, w.chunks, w.rank, w.rec));
            CUDA_TRY(w.chunk_items.alloc((size_t)B * 32));
            CUDA_TRY(alloc_each(nt, w.tcount, w.tbase));
            CUDA_TRY(cudaMemset(w.tcount.get(), 0, sizeof(int32_t) * nt));
        }
        e->win_ready = true;
    }
    return RAMP_OK;
}

void launch_step_kernel(ramp_engine* e, const ramp_action_t* d_actions, int32_t fuse, double* d_stats_out, int32_t* d_ncs_out) {
    const int B = e->cfg.n_episodes;
    StepArgs s{};
    s.actions = d_actions; s.ep = e->ep; s.res = e->res.view(); s.pool = e->pool.view(); s.counters = e->d_counters.get();
    s.stats_out = d_stats_out; s.n_cluster_steps_out = d_ncs_out; s.fuse_empty_steps = fuse;
    step_kernel_for(e->step_nt)<<<(B + e->step_nt - 1) / e->step_nt, e->step_nt, e->step_smem, e->stream.get()>>>(s);
    e->launches++;
}

// One step whose lookaheads may run while the steps before it are still running (DESIGN.md §4):
//   plan stream     speculative plan (actions read ahead of the step), bucket
//   window stream   thread kernel
//   engine stream   commit (the exact plan, in stream order), repair bucket + thread kernel (lookaheads the speculative plan
//                   missed because the actions changed after it read them; normally none), step kernel
int step_overlapped(ramp_engine* e, const ramp_action_t* d_actions, int32_t fuse, double* d_stats_out, int32_t* d_ncs_out) {
    int rc = ensure_windows(e);
    if (rc != RAMP_OK) return rc;
    const int B = e->cfg.n_episodes, grid_b = (B + 127) / 128;
    const int32_t n_templates = (int32_t)e->templates.size();
    LookaheadWindow& w = e->win[e->win_seq++ % N_WINDOWS];
    cudaStream_t ps = e->plan_stream.get(), ws = w.stream.get(), st = e->stream.get();
    if (e->ev_pending >= MAX_EVENT_PAIRS) { CUDA_TRY(cudaStreamSynchronize(st)); rc = resolve_events(e); if (rc) return rc; }
    CUDA_TRY(cudaStreamWaitEvent(ps, w.ev_consumed.get(), 0));
    if (e->reset_pending) { CUDA_TRY(cudaStreamWaitEvent(ps, e->ev_reset.get(), 0)); e->reset_pending = false; }
    SpecPlanArgs sp{};
    sp.actions = d_actions; sp.templates = e->d_templates.get(); sp.n_templates = n_templates; sp.B = B;
    sp.keys = e->d_spec_keys.get(); sp.mask = e->memo_cap - 1; sp.slot_base = e->spec_base;
    sp.items_res = w.items_res.get(); sp.counters = w.counters.get(); sp.rec = w.rec.get();
    ramp_spec_plan_kernel<<<grid_b, 128, 0, ps>>>(sp);
    CUDA_TRY(cudaEventRecord(e->ev_a[e->ev_pending].get(), ps));
    bucket_resident(e, w.items_res.get(), w.counters.get(), w.chunk_items.get(), w.chunks.get(), w.rank.get(), w.tcount.get(), w.tbase.get(), ps);
    CUDA_TRY(cudaEventRecord(w.ev_planned.get(), ps));
    CUDA_TRY(cudaStreamWaitEvent(ws, w.ev_planned.get(), 0));
    ThreadArgs ta = make_thread_args(e, w.chunks.get(), w.chunk_items.get(), w.counters.get(), e->res.view(), e->pool.view(), e->d_stats.get());
    ramp_lookahead_thread_kernel<<<e->res_grid, RAMP_THREAD_CTA, e->res_smem, ws>>>(ta);
    CUDA_TRY(cudaEventRecord(e->ev_b[e->ev_pending].get(), ws));
    e->ev_pending++;
    CUDA_TRY(cudaEventRecord(w.ev_end.get(), ws));
    CUDA_TRY(cudaStreamWaitEvent(st, w.ev_end.get(), 0));
    CommitArgs c{};
    c.actions = d_actions; c.templates = e->d_templates.get(); c.n_templates = n_templates; c.ep = e->ep;
    c.memo.keys = e->d_memo_keys.get(); c.memo.mask = e->memo_cap - 1; c.memo.mode = e->cfg.memo_mode; c.memo.vals = e->d_memo_vals.get();
    c.rec = w.rec.get(); c.repair_keys = e->d_repair_keys.get(); c.repair_mask = e->memo_cap - 1; c.repair_base = e->repair_base;
    c.items_res = w.items_res.get(); c.win_counters = w.counters.get(); c.counters = e->d_counters.get(); c.stats = e->d_stats.get();
    ramp_commit_kernel<<<grid_b, 128, 0, st>>>(c);
    bucket_resident(e, w.items_res.get(), w.counters.get(), w.chunk_items.get(), w.chunks.get(), w.rank.get(), w.tcount.get(), w.tbase.get(), st);
    ramp_lookahead_thread_kernel<<<e->res_grid, RAMP_THREAD_CTA, e->res_smem, st>>>(ta);   // the repair launch: usually no chunk
    CUDA_TRY(cudaEventRecord(w.ev_consumed.get(), st));
    launch_step_kernel(e, d_actions, fuse, d_stats_out, d_ncs_out);
    e->launches += 4;
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

}  // namespace

// hooks for the other translation units of the library (ramp_policy.cu); not part of the C ABI
int ramp_internal_set_error(int code, const char* msg) { g_last_error = msg; return code; }
cudaStream_t ramp_internal_stream(ramp_engine_t* e) { return e->stream.get(); }
int ramp_internal_device(ramp_engine_t* e) { return e->cfg.device; }
void ramp_internal_count_launches(ramp_engine_t* e, int n) { e->launches += n; }
// the device environment's per-episode return and env-step count (ramp_es_*); RAMP_ERR_BAD_ARG without an environment
int ramp_internal_env_returns(ramp_engine_t* e, const double** ret, const int32_t** n_decided) {
    if (!e || !e->has_env) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    *ret = e->env.ret;
    *n_decided = e->env.n_decided;
    return RAMP_OK;
}

extern "C" {

const char* ramp_last_error(void) { return g_last_error.c_str(); }

#ifdef RAMP_TICK_CLOCKS
// measurement builds only (scripts/tick_cycles.py): the thread kernel's cycle ledger summed over CTAs into
// out[RAMP_TC_SHAPES][RAMP_TC_PHASES + 1] (cycles per phase, then ticks), on the current device; reset = 1 zeroes it after
int ramp_debug_tick_clocks(unsigned long long* out, int reset) {
    static unsigned long long h[RAMP_TC_MAX_CTAS][RAMP_TC_SHAPES][RAMP_TC_PHASES + 1];
    CUDA_TRY(cudaDeviceSynchronize());
    CUDA_TRY(cudaMemcpyFromSymbol(h, ramp::ramp_tick_clocks, sizeof(h)));
    memset(out, 0, sizeof(h[0]));
    for (int b = 0; b < RAMP_TC_MAX_CTAS; ++b)
        for (int s = 0; s < RAMP_TC_SHAPES; ++s)
            for (int i = 0; i <= RAMP_TC_PHASES; ++i) out[s * (RAMP_TC_PHASES + 1) + i] += h[b][s][i];
    if (reset) { memset(h, 0, sizeof(h)); CUDA_TRY(cudaMemcpyToSymbol(ramp::ramp_tick_clocks, h, sizeof(h))); }
    return RAMP_OK;
}
#endif

int ramp_engine_create(const ramp_config_t* cfg_in, ramp_engine_t** out) {
    if (!cfg_in || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    ramp_config_t cfg = *cfg_in;
    if (cfg.n_episodes < 1 || cfg.max_jobs < 1 || cfg.n_cluster_workers < 1)
        return set_error(RAMP_ERR_BAD_ARG, "n_episodes, max_jobs and n_cluster_workers must be >= 1");
    if (cfg.max_running < 1) cfg.max_running = cfg.n_cluster_workers;
    if (cfg.max_templates < 1) cfg.max_templates = 1024;
    if (cfg.trace_cap < 1) cfg.trace_cap = 16384;
    if (cfg.job_queue_capacity < 0) cfg.job_queue_capacity = 10;
    if (cfg.machine_epsilon == 0.0) cfg.machine_epsilon = 1e-7;
    if (cfg.memo_capacity_log2 <= 0) {
        int lg = 10;
        while ((1ll << lg) < (long long)cfg.n_episodes * 16 && lg < 26) ++lg;
        cfg.memo_capacity_log2 = lg;
    }
    CUDA_TRY(cudaSetDevice(cfg.device));
    std::unique_ptr<ramp_engine> e(new ramp_engine());     // frees whatever was allocated when a step below fails
    e->cfg = cfg;
    if (const char* v = getenv("RAMP_LOOKAHEAD_CTA_THREADS")) {
        const int nt = atoi(v);
        if (lookahead_cta_kernel_for(nt) == nullptr) return set_error(RAMP_ERR_BAD_ARG, "RAMP_LOOKAHEAD_CTA_THREADS must be 64, 128 or 256");
        e->cta_nt = nt;
    }
    if (const char* v = getenv("RAMP_LOOKAHEAD_MODE")) {
        // auto (or thread): resident whenever the quotient blob fits; cta: every template on the CTA kernel (no resident
        // quotient blobs); thread_unfolded: the thread kernel on the unfolded job (identity quotient)
        if (!strcmp(v, "cta")) e->cta_only = true;
        else if (!strcmp(v, "thread_unfolded")) e->use_quotient = 0;
        else if (strcmp(v, "auto") != 0 && strcmp(v, "thread") != 0)
            return set_error(RAMP_ERR_BAD_ARG, "RAMP_LOOKAHEAD_MODE must be auto, thread, thread_unfolded or cta, not '%s'", v);
    }
    if (const char* v = getenv("RAMP_DEBUG")) e->debug = atoi(v);
    if (const char* v = getenv("RAMP_STEP_OVERLAP")) e->overlap = atoi(v) != 0;   // 0: the in-order path only (tests compare the two)
    cudaDeviceProp prop{};
    CUDA_TRY(cudaGetDeviceProperties(&prop, cfg.device));
    e->sm_count = prop.multiProcessorCount;
    CUDA_TRY(create(e->stream, cudaStreamNonBlocking));
    const int B = cfg.n_episodes;

    CUDA_TRY(e->d_templates.alloc(cfg.max_templates));
    e->memo_cap = 1u << cfg.memo_capacity_log2;
    CUDA_TRY(e->d_memo_keys.alloc(e->memo_cap));
    CUDA_TRY(cudaMemset(e->d_memo_keys.get(), 0, sizeof(unsigned long long) * e->memo_cap));
    CUDA_TRY(e->d_memo_vals.alloc(e->memo_cap));
    e->memo_cap2 = 1;
    while (e->memo_cap2 < (uint32_t)cfg.max_templates * 2u) e->memo_cap2 <<= 1;
    CUDA_TRY(e->d_memo_keys2.alloc(e->memo_cap2));
    CUDA_TRY(cudaMemset(e->d_memo_keys2.get(), 0, sizeof(unsigned long long) * e->memo_cap2));
    // slots: the memo's positions, B for RAMP_MEMO_OFF, the level-2 cache, then the result and repair tables of overlapped steps
    e->spec_base = (int32_t)e->memo_cap + B + (int32_t)e->memo_cap2;
    e->repair_base = e->spec_base + (int32_t)e->memo_cap;
    e->n_slots = e->repair_base + (int32_t)e->memo_cap;
    CUDA_TRY(alloc_each(e->memo_cap, e->d_spec_keys, e->d_repair_keys));
    CUDA_TRY(cudaMemset(e->d_spec_keys.get(), 0, sizeof(unsigned long long) * e->memo_cap));
    CUDA_TRY(cudaMemset(e->d_repair_keys.get(), 0, sizeof(unsigned long long) * e->memo_cap));
    CUDA_TRY(e->res.alloc(e->n_slots));
    CUDA_TRY(cudaMemset(e->res.status.get(), 0, sizeof(int32_t) * e->n_slots));

    // trace pool: exact-size allocations; 4 Mi entries at least, else enough for 8 un-memoised lookaheads of 2,048 ticks per
    // episode between two resets (the pool is reset with the memo)
    CUDA_TRY(e->pool.alloc(std::max<uint64_t>(4ull << 20, (uint64_t)B * 8ull * 2048ull)));      // B=1: 48 MiB; B=4096: 805 MiB
    CUDA_TRY(cudaMemset(e->pool.top.get(), 0, sizeof(unsigned long long)));

    CUDA_TRY(alloc_each(B, e->d_items, e->d_items_res, e->d_chunks, e->d_rank, e->d_actions, e->d_n_cluster_steps));
    CUDA_TRY(e->d_chunk_items.alloc((size_t)B * 32));
    CUDA_TRY(alloc_each((size_t)cfg.max_templates + 1, e->d_tcount, e->d_tbase));
    CUDA_TRY(cudaMemset(e->d_tcount.get(), 0, sizeof(int32_t) * ((size_t)cfg.max_templates + 1)));
    CUDA_TRY(e->d_hints.alloc(cfg.max_templates));
    CUDA_TRY(cudaMemset(e->d_hints.get(), 0, sizeof(TemplateHints) * (size_t)cfg.max_templates));
    CUDA_TRY(e->d_hint_jct.alloc(cfg.max_templates));
    CUDA_TRY(cudaMemset(e->d_hint_jct.get(), 0, sizeof(double) * (size_t)cfg.max_templates));
    CUDA_TRY(e->d_counters.alloc(1));
    CUDA_TRY(e->d_stats.alloc(2));
    CUDA_TRY(cudaMemset(e->d_counters.get(), 0, sizeof(Counters)));
    CUDA_TRY(cudaMemset(e->d_stats.get(), 0, 2 * sizeof(MemoStats)));
    CUDA_TRY(e->d_step_stats.alloc((size_t)RAMP_STEP_STATS_LEN * B));
    CUDA_TRY(e->d_ep_export.alloc((size_t)RAMP_EP_LEN * B));
    CUDA_TRY(e->d_es_export.alloc((size_t)RAMP_ES_LEN * B));
    CUDA_TRY(e->h_n_work.alloc(1));
    CUDA_TRY(e->h_stats.alloc(2));

    EpisodeState& ep = e->ep;
    ep.B = B; ep.max_running = cfg.max_running; ep.max_jobs = cfg.max_jobs; ep.n_jobs = 0;
    ep.n_cluster_workers = cfg.n_cluster_workers; ep.queue_capacity = cfg.job_queue_capacity;
    ep.eps = cfg.machine_epsilon; ep.max_sim_time = cfg.max_simulation_run_time;
    CUDA_TRY(e->ep_ef.alloc((size_t)EF_COUNT * B));
    CUDA_TRY(e->ep_ei.alloc((size_t)EI_COUNT * B));
    CUDA_TRY(e->ep_rf.alloc((size_t)RF_COUNT * cfg.max_running * B));
    CUDA_TRY(e->ep_ri.alloc((size_t)RI_COUNT * cfg.max_running * B));
    CUDA_TRY(e->ep_rec.alloc((size_t)cfg.max_jobs * B));
    CUDA_TRY(e->d_arrivals.alloc((size_t)cfg.max_jobs * B));
    CUDA_TRY(e->h_arr_stage.alloc((size_t)cfg.max_jobs * B));
    CUDA_TRY(create(e->ev_stage, cudaEventDisableTiming));
    ep.ef = e->ep_ef.get(); ep.ei = e->ep_ei.get(); ep.rf = e->ep_rf.get(); ep.ri = e->ep_ri.get(); ep.rec = e->ep_rec.get();
    CUDA_TRY(cudaMemset(ep.ef, 0, sizeof(double) * EF_COUNT * B));
    CUDA_TRY(cudaMemset(ep.ei, 0, sizeof(int32_t) * EI_COUNT * B));
    CUDA_TRY(cudaMemset(ep.rec, 0, sizeof(ramp_job_record_t) * (size_t)cfg.max_jobs * B));
    ep.arr = e->d_arrivals.get();
    CUDA_TRY(e->d_n_jobs_ep.alloc(B));
    CUDA_TRY(cudaMemset(e->d_n_jobs_ep.get(), 0, sizeof(int32_t) * B));
    ep.n_jobs_ep = e->d_n_jobs_ep.get();
    // 32 episodes per CTA puts 4,096 episodes on 128 SMs; a table too large for 32 copies in shared memory takes one per CTA
    {
        const int rows = step_rows(cfg.max_running, cfg.max_jobs);
        e->step_nt = step_smem_bytes(32, rows) <= STEP_SMEM_MAX ? 32 : 1;
        e->step_smem = step_smem_bytes(e->step_nt, rows);
        if (e->step_smem > STEP_SMEM_MAX)
            return set_error(RAMP_ERR_CAPACITY, "the running-job table of %d rows needs %zu B of shared memory (max %zu)", rows, e->step_smem,
                             (size_t)STEP_SMEM_MAX);
        CUDA_TRY(reserve_dynamic_smem((const void*)step_kernel_for(e->step_nt), e->step_smem));
    }

    for (int k = 0; k < MAX_EVENT_PAIRS; ++k) {
        CUDA_TRY(create(e->ev_a[k], cudaEventDefault));
        CUDA_TRY(create(e->ev_b[k], cudaEventDefault));
    }
    *out = e.release();
    return RAMP_OK;
}

int ramp_engine_destroy(ramp_engine_t* e) {
    if (!e) return RAMP_OK;
    cudaSetDevice(e->cfg.device);
    cudaStreamSynchronize(e->stream.get());
    if (e->win_ready) {
        cudaStreamSynchronize(e->plan_stream.get());
        for (LookaheadWindow& w : e->win) cudaStreamSynchronize(w.stream.get());
    }
    delete e;
    return RAMP_OK;
}

void* ramp_engine_stream(ramp_engine_t* e) { return e ? (void*)e->stream.get() : nullptr; }

int ramp_template_count(ramp_engine_t* e) { return e ? (int)e->templates.size() : 0; }

int ramp_register_template(ramp_engine_t* e, const ramp_lowered_job_t* j, int32_t* id_out) {
    if (!e || !j || !id_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    // a captured step's graph holds the template count and the lookahead scratch that registering a template may change
    if (e->env_captured)
        return set_error(RAMP_ERR_BAD_ARG, "no template can be registered once a step was captured into a CUDA graph: the graph keeps "
                         "the template count and the lookahead scratch a new template may regrow");
    if ((int)e->templates.size() >= e->cfg.max_templates)
        return set_error(RAMP_ERR_CAPACITY, "max_templates (%d) reached", e->cfg.max_templates);
    const int32_t N = j->n_ops, E = j->n_deps, W = j->n_workers, C = j->n_channels;
    if (N < 1 || E < 0 || W < 1 || C < 0) return set_error(RAMP_ERR_BAD_ARG, "bad template sizes N=%d E=%d W=%d C=%d", N, E, W, C);
    if (W > 0xFFFF || C >= 0xFFFF) return set_error(RAMP_ERR_BAD_ARG, "too many mounted workers/channels");
    if (j->model_id < 0 || j->model_id > 0xFFFF || j->degree < 0 || j->degree > 0xFFFF)
        return set_error(RAMP_ERR_BAD_ARG, "model_id and degree must fit 16 bits");
    // ---- validate (the reference would KeyError / misbehave on these) ----
    if (j->row_ptr[0] != 0 || j->row_ptr[N] != E) return set_error(RAMP_ERR_BAD_ARG, "row_ptr is not a CSR offset array");
    for (int32_t i = 0; i < N; ++i) {
        if (j->row_ptr[i + 1] < j->row_ptr[i]) return set_error(RAMP_ERR_BAD_ARG, "row_ptr not monotone at %d", i);
        if (j->op_worker[i] >= W) return set_error(RAMP_ERR_BAD_ARG, "op %d on worker %d >= n_workers %d", i, j->op_worker[i], W);
        if (!(j->op_cost[i] >= 0.0)) return set_error(RAMP_ERR_BAD_ARG, "op %d has a negative or NaN cost", i);
    }
    std::vector<int32_t> in_deg(N, 0);
    for (int32_t k = 0; k < E; ++k) {
        if (j->dep_dst[k] < 0 || j->dep_dst[k] >= N) return set_error(RAMP_ERR_BAD_ARG, "dep %d has dst out of range", k);
        if (j->dep_channel[k] != RAMP_NO_CHANNEL && j->dep_channel[k] >= C)
            return set_error(RAMP_ERR_BAD_ARG, "dep %d on channel %d >= n_channels %d", k, j->dep_channel[k], C);
        if (!(j->dep_run_time[k] >= 0.0)) return set_error(RAMP_ERR_BAD_ARG, "dep %d has a negative or NaN run time", k);
        // RCE:542-560 zeroes the run time of every non-flow dep when the job is mounted; with a non-zero one the reference's
        // zero-length ticks (RCE:412-422) would never complete it and _run_lookahead would spin forever
        if (!j->dep_is_flow[k] && j->dep_run_time[k] != 0.0)
            return set_error(RAMP_ERR_BAD_ARG, "non-flow dep %d has a non-zero run time (RCE:542-560 zeroes it)", k);
        in_deg[j->dep_dst[k]]++;
    }
    for (int32_t i = 0; i < N; ++i)
        if ((int32_t)j->op_n_parents[i] > in_deg[i])
            return set_error(RAMP_ERR_BAD_ARG, "op %d has n_parents %d > in-degree %d", i, (int)j->op_n_parents[i], in_deg[i]);
    // ---- derive ----
    std::vector<uint32_t> op_key, dep_key;
    make_rank_keys(j->op_prio, N, op_key);
    make_rank_keys(j->dep_prio, E, dep_key);
    std::vector<int32_t> src;
    for (int32_t i = 0; i < N; ++i) if (in_deg[i] == 0) src.push_back(i);
    std::vector<double> op_cost(j->op_cost, j->op_cost + N), dep_rt(j->dep_run_time, j->dep_run_time + E);
    for (auto& x : op_cost) x = x + 0.0;   // -0.0 -> +0.0 so the u64 bit pattern orders like the value
    for (auto& x : dep_rt) x = x + 0.0;

    // ---- records in the layout the tick loop streams (see TemplateDev) ----
    struct OpRec { double cost; uint32_t key; uint32_t worker; };
    static_assert(sizeof(OpRec) == 16, "op record must be 16 bytes");
    std::vector<OpRec> op_rec(N);
    std::vector<int32_t> op_row((size_t)N * 2, 0);
    for (int32_t i = 0; i < N; ++i) {
        op_rec[i] = OpRec{op_cost[i], op_key[i], (uint32_t)j->op_worker[i]};
        op_row[(size_t)i * 2] = j->row_ptr[i];
        op_row[(size_t)i * 2 + 1] = j->row_ptr[i + 1] - j->row_ptr[i];
    }
    int32_t max_in_deg = 0;
    for (int32_t i = 0; i < N; ++i) max_in_deg = std::max(max_in_deg, in_deg[i]);
    const bool par_in_smem = (max_in_deg <= 255 && N <= 8192);       // byte parent counters in shared memory
    // the whole dep in one word for the kernels' 16-byte frontier entries (TemplateDev::dep_kd)
    auto bits_for = [](uint64_t max_value) { int b = 1; while ((max_value >> b) != 0) ++b; return b; };
    const int kbits = bits_for((uint64_t)std::max(E, 1));                 // keys are 1..E, 0 = "none"
    const int cbits = bits_for((uint64_t)C + 1);                          // channels 0..C-1, all ones = "none"
    const int nbits = bits_for((uint64_t)N);
    if (kbits + cbits + 9 + nbits > 64)
        return set_error(RAMP_ERR_CAPACITY, "template too large for the packed dep word: %d key + %d channel + 9 + %d op bits > 64",
                         kbits, cbits, nbits);
    const uint32_t kd_kmask = (uint32_t)((1ull << kbits) - 1ull), kd_cmask = (uint32_t)((1ull << cbits) - 1ull);
    const int kd_cshift = kbits, kd_fshift = kbits + cbits, kd_dshift = kbits + cbits + 9;
    std::vector<unsigned long long> dep_kd(E);
    for (int32_t k = 0; k < E; ++k) {
        const unsigned long long chan = (j->dep_channel[k] == RAMP_NO_CHANNEL) ? (unsigned long long)kd_cmask : (unsigned long long)j->dep_channel[k];
        dep_kd[k] = (unsigned long long)dep_key[k] | (chan << kd_cshift)
                    | ((unsigned long long)(j->dep_is_flow[k] ? 1 : 0) << kd_fshift)
                    | (par_in_smem ? ((unsigned long long)j->op_n_parents[j->dep_dst[k]] << (kd_fshift + 1)) : 0ull)
                    | ((unsigned long long)j->dep_dst[k] << kd_dshift);
    }

    // ---- pack one blob ----
    struct Seg { const void* p; size_t bytes; size_t off; };
    Seg segs[6] = {
        {op_rec.data(), sizeof(OpRec) * (size_t)N, 0}, {j->op_n_parents, sizeof(uint16_t) * (size_t)N, 0},
        {op_row.data(), sizeof(int32_t) * op_row.size(), 0}, {dep_kd.data(), sizeof(unsigned long long) * (size_t)E, 0},
        {dep_rt.data(), sizeof(double) * (size_t)E, 0}, {src.data(), sizeof(int32_t) * src.size(), 0}};
    size_t total = 0;
    for (auto& s : segs) { s.off = total; total += align_up(std::max<size_t>(s.bytes, 1), 256); }
    HostTemplate ht;
    ht.bytes.assign(total + 8 * sizeof(int32_t), 0);
    for (auto& s : segs) if (s.bytes) memcpy(ht.bytes.data() + s.off, s.p, s.bytes);
    int32_t hdr[8] = {N, E, W, C, j->num_training_steps, 0, 0, (int32_t)src.size()};
    memcpy(ht.bytes.data() + total, hdr, sizeof(hdr));
    ht.hash = fnv1a(ht.bytes.data(), ht.bytes.size());
    int32_t canon = (int32_t)e->templates.size();
    for (size_t t = 0; t < e->templates.size(); ++t)
        if (e->templates[t].hash == ht.hash && e->templates[t].bytes == ht.bytes) { canon = e->templates[t].dev.canon_id; break; }

    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(ht.blob.alloc(total));
    CUDA_TRY(cudaMemcpy(ht.blob.get(), ht.bytes.data(), total, cudaMemcpyHostToDevice));
    unsigned char* base = ht.blob.get();
    TemplateDev& d = ht.dev;
    d.n_ops = N; d.n_deps = E; d.n_workers = W; d.n_channels = C;
    d.num_training_steps = j->num_training_steps; d.model_id = j->model_id; d.degree = j->degree;
    d.n_src = (int32_t)src.size(); d.canon_id = canon;
    d.size_class = 0;
    d.par_in_smem = par_in_smem ? 1 : 0;
    d._pad0 = 0;
    d.op_rec = (const int4*)(base + segs[0].off); d.op_n_parents = (const uint16_t*)(base + segs[1].off);
    d.op_row = (const int2*)(base + segs[2].off); d.dep_kd = (const unsigned long long*)(base + segs[3].off);
    d.dep_rt = (const double*)(base + segs[4].off); d.src_ops = (const int32_t*)(base + segs[5].off);
    d.kd_kmask = kd_kmask; d.kd_cmask = kd_cmask; d.kd_cshift = kd_cshift; d.kd_fshift = kd_fshift; d.kd_dshift = kd_dshift; d._pad1 = 0;
    d.scratch_bytes = scratch_bytes_for(N, E);
    d.algorithmic_bytes_static = 20ull * (uint64_t)N + 19ull * (uint64_t)E + 24ull;
    // ---- symmetry quotient -> resident blob for the thread-per-lookahead kernel ----
    d.res_blob = nullptr; d.res_bytes = 0; d.res_n_ops = 0; d.res_n_deps = 0; d._pad2 = 0;
    if (!e->cta_only) {
        ramp_quotient_t q{};
        const int qrc = e->use_quotient ? ramp_quotient_template(j, &q) : identity_quotient(j, &q);
        if (qrc != RAMP_OK) return set_error(qrc, "ramp_quotient_template failed (%d)", qrc);
        std::vector<unsigned char> rblob;
        if (build_resident_blob(j, q, RESIDENT_MAX_BYTES, rblob)) {
            cudaError_t ce = ht.res_blob.alloc(rblob.size());
            if (ce == cudaSuccess) ce = cudaMemcpy(ht.res_blob.get(), rblob.data(), rblob.size(), cudaMemcpyHostToDevice);
            if (ce != cudaSuccess) { ramp_free_quotient(&q); return set_error(RAMP_ERR_CUDA, "resident blob upload failed: %s", cudaGetErrorString(ce)); }
            d.res_blob = ht.res_blob.get(); d.res_bytes = (int32_t)rblob.size();
            d.res_n_ops = q.n_ops; d.res_n_deps = q.n_deps;
            d.size_class = 2;
            e->res_tmpl_cap = std::max(e->res_tmpl_cap, (int32_t)align_up((uint64_t)rblob.size(), 128));
            e->res_n_cap = std::max(e->res_n_cap, (int32_t)align_up((uint64_t)q.n_ops, 2));
            e->res_spill_ops = std::max(e->res_spill_ops, q.n_ops);
            e->res_spill_deps = std::max(e->res_spill_deps, std::max(q.n_deps, 1));
        }
        if (e->debug) fprintf(stderr, "[ramp] template %d: N=%d E=%d W=%d C=%d -> quotient N=%d E=%d W=%d C=%d, %s (%zu B)\n", (int)e->templates.size(),
                              N, E, W, C, q.n_ops, q.n_deps, q.n_workers, q.n_channels, d.res_blob ? "resident" : "not resident", rblob.size());
        ramp_free_quotient(&q);
    }
    const int32_t id = (int32_t)e->templates.size();
    CUDA_TRY(cudaMemcpy(e->d_templates.get() + id, &d, sizeof(TemplateDev), cudaMemcpyHostToDevice));
    if (d.size_class == 2) e->n_resident++; else e->n_nonresident++;
    if (d.size_class != 2) {       // the CTA kernel's slabs and shared-memory tables are sized by the jobs that use them
        e->max_scratch = std::max(e->max_scratch, d.scratch_bytes);
        e->max_w = std::max(e->max_w, W);
        e->max_c = std::max(e->max_c, std::max(C, 1));
        if (d.par_in_smem) e->par_cap = std::max(e->par_cap, (int32_t)align_up((uint64_t)N, 16));
    }
    e->templates.push_back(std::move(ht));
    *id_out = id;
    return RAMP_OK;
}

int ramp_reset(ramp_engine_t* e, const ramp_arrival_t* arrivals, int32_t n_jobs) {
    if (!e || !arrivals) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (n_jobs < 1 || n_jobs > e->cfg.max_jobs) return set_error(RAMP_ERR_BAD_ARG, "n_jobs %d not in [1, max_jobs=%d]", n_jobs, e->cfg.max_jobs);
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    const int B = e->cfg.n_episodes;
    cudaStream_t st = e->stream.get();
    // the caller may overwrite `arrivals` as soon as this returns, so they are copied into the pinned staging buffer (once the
    // previous reset's upload from it has finished) and uploaded from there in stream order; nothing here waits for the device
    CUDA_TRY(cudaEventSynchronize(e->ev_stage.get()));
    const size_t row = sizeof(ramp_arrival_t) * (size_t)n_jobs;
    memcpy(e->h_arr_stage.get(), arrivals, row * B);
    if (n_jobs == e->cfg.max_jobs) {
        CUDA_TRY(cudaMemcpyAsync(e->d_arrivals.get(), e->h_arr_stage.get(), row * B, cudaMemcpyHostToDevice, st));
    } else {
        CUDA_TRY(cudaMemcpy2DAsync(e->d_arrivals.get(), sizeof(ramp_arrival_t) * (size_t)e->cfg.max_jobs, e->h_arr_stage.get(), row, row, B,
                                   cudaMemcpyHostToDevice, st));
    }
    CUDA_TRY(cudaEventRecord(e->ev_stage.get(), st));
    e->ep.n_jobs = n_jobs;
    // memo is per env instance per episode: cleared on reset (RCE:269-275)
    CUDA_TRY(cudaMemsetAsync(e->d_memo_keys.get(), 0, sizeof(unsigned long long) * e->memo_cap, st));
    if (e->win_ready) {
        // every window of an enqueued step ends before that step's step kernel, so these clears come after all of them; the
        // next speculative plan waits for them
        CUDA_TRY(cudaMemsetAsync(e->d_spec_keys.get(), 0, sizeof(unsigned long long) * e->memo_cap, st));
        CUDA_TRY(cudaMemsetAsync(e->d_repair_keys.get(), 0, sizeof(unsigned long long) * e->memo_cap, st));
    }
    // the batch-wide cache of RAMP_MEMO_SHARED (level-2 keys, its result slots and traces) is a pure function of the
    // lowered job and survives the reset; every other mode starts from an empty trace pool
    if (e->cfg.memo_mode != RAMP_MEMO_SHARED) CUDA_TRY(cudaMemsetAsync(e->pool.top.get(), 0, sizeof(unsigned long long), st));
    // the counters stay cumulative; memo statistics are reported since this copy of them
    CUDA_TRY(cudaMemcpyAsync(e->d_stats.get() + 1, e->d_stats.get(), sizeof(MemoStats), cudaMemcpyDeviceToDevice, st));
    CUDA_TRY(cudaMemsetAsync(e->d_counters.get(), 0, sizeof(Counters), st));
    ramp_reset_kernel<<<(B + 127) / 128, 128, 0, st>>>(e->ep, e->d_n_jobs_ep.get(), n_jobs);
    e->launches++;
    if (e->win_ready) { CUDA_TRY(cudaEventRecord(e->ev_reset.get(), st)); e->reset_pending = true; }
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

int ramp_set_arrivals(ramp_engine_t* e, int32_t episode, int32_t first_job, const ramp_arrival_t* rows, int32_t n) {
    if (!e || !rows) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (episode < 0 || episode >= e->cfg.n_episodes || first_job < 0 || n < 0 || first_job + n > e->cfg.max_jobs)
        return set_error(RAMP_ERR_BAD_ARG, "arrival rows [%d, %d) of episode %d out of range (max_jobs=%d)", first_job, first_job + n, episode, e->cfg.max_jobs);
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaMemcpyAsync(e->d_arrivals.get() + (size_t)episode * e->cfg.max_jobs + first_job, rows, sizeof(ramp_arrival_t) * (size_t)n,
                             cudaMemcpyHostToDevice, e->stream.get()));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    return RAMP_OK;
}

int ramp_set_job_count(ramp_engine_t* e, int32_t episode, int32_t n_jobs) {
    if (!e) return set_error(RAMP_ERR_BAD_ARG, "null engine");
    if (episode < 0 || episode >= e->cfg.n_episodes || n_jobs < 0 || n_jobs > e->cfg.max_jobs)
        return set_error(n_jobs > e->cfg.max_jobs ? RAMP_ERR_CAPACITY : RAMP_ERR_BAD_ARG,
                         "job count %d of episode %d out of range (max_jobs=%d)", n_jobs, episode, e->cfg.max_jobs);
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaMemcpyAsync(e->d_n_jobs_ep.get() + episode, &n_jobs, sizeof(int32_t), cudaMemcpyHostToDevice, e->stream.get()));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    return RAMP_OK;
}

int ramp_set_limits(ramp_engine_t* e, double max_sim_time, int32_t queue_capacity) {
    if (!e) return set_error(RAMP_ERR_BAD_ARG, "null engine");
    if (queue_capacity < 0 || !(max_sim_time > 0.0)) return set_error(RAMP_ERR_BAD_ARG, "bad limits");
    e->cfg.max_simulation_run_time = max_sim_time; e->cfg.job_queue_capacity = queue_capacity;
    e->ep.max_sim_time = max_sim_time; e->ep.queue_capacity = queue_capacity;
    return RAMP_OK;
}

int ramp_step_device(ramp_engine_t* e, const ramp_action_t* d_actions, int32_t fuse, double* d_stats_out, int32_t* d_ncs_out) {
    if (!e || !d_actions) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (e->ep.n_jobs < 1) return set_error(RAMP_ERR_BAD_ARG, "ramp_reset must be called before ramp_step");
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    cudaStream_t st = e->stream.get();
    // under capture (the engine stream forked into a caller's capture) the buffers are those the last eager step sized, and the
    // step neither times itself nor reads anything back
    bool capturing = false;
    int rc0 = capture_status(st, &capturing);
    if (rc0 == RAMP_OK && capturing) rc0 = capture_refusal(e);
    if (rc0 != RAMP_OK) return rc0;
    if (!capturing) {
        if (e->n_nonresident > 0) { int rc = ensure_scratch(e); if (rc != RAMP_OK) return rc; }
        if (e->n_resident > 0) { int rc = ensure_thread_scratch(e); if (rc != RAMP_OK) return rc; }
        e->sized_templates = (int64_t)e->templates.size();
    }
    // the overlapped path covers per-episode memo keys on resident templates; steps with engine-written actions, a template
    // on the CTA kernel (its launch shape needs the work count on the host), another memo mode or a capture run in order
    if (e->overlap && e->cfg.memo_mode == RAMP_MEMO_REFERENCE && e->n_nonresident == 0 && e->n_resident > 0 && !engine_owned(e, d_actions) &&
        !capturing)
        return step_overlapped(e, d_actions, fuse, d_stats_out, d_ncs_out);
    const int B = e->cfg.n_episodes;
    CUDA_TRY(cudaMemsetAsync(e->d_counters.get(), 0, 2 * sizeof(int32_t), st));   // n_work and work_cursor
    PlanArgs p{};
    p.actions = d_actions; p.templates = e->d_templates.get(); p.n_templates = (int32_t)e->templates.size();
    p.ep = e->ep; p.memo.keys = e->d_memo_keys.get(); p.memo.mask = e->memo_cap - 1; p.memo.mode = e->cfg.memo_mode;
    p.memo.vals = e->d_memo_vals.get(); p.memo.keys2 = e->d_memo_keys2.get(); p.memo.mask2 = e->memo_cap2 - 1;
    p.memo.slot2_base = (int32_t)e->memo_cap + e->cfg.n_episodes;
    p.items = e->d_items.get(); p.items_res = e->d_items_res.get(); p.counters = e->d_counters.get(); p.stats = e->d_stats.get();
    ramp_plan_kernel<<<(B + 127) / 128, 128, 0, st>>>(p);
    e->launches++;
    if (!e->templates.empty()) {
        if (!capturing) {                // a replay would record the pair again with no host to resolve it
            if (e->ev_pending >= MAX_EVENT_PAIRS) { CUDA_TRY(cudaStreamSynchronize(st)); int rc = resolve_events(e); if (rc) return rc; }
            CUDA_TRY(cudaEventRecord(e->ev_a[e->ev_pending].get(), st));
        }
        // memo misses on resident templates: one THREAD per lookahead, grouped on the device.  Their count stays there: idle
        // CTAs find the chunk cursor exhausted and exit.
        if (e->n_resident > 0) bucket_resident(e, e->d_items_res.get(), e->d_counters.get(), e->d_chunk_items.get(), e->d_chunks.get(), e->d_rank.get(),
                                        e->d_tcount.get(), e->d_tbase.get(), st);
        int n_nonres = 0;
        if (e->n_nonresident > 0) {
            // the number of memo misses on non-resident templates decides the CTA kernel's shape: a 4-byte read-back (~10 us)
            // against multi-ms kernels
            CUDA_TRY(cudaMemcpyAsync(e->h_n_work.get(), &e->d_counters.get()->n_work, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            n_nonres = e->h_n_work.get()[0];
        }
        int rc = launch_lookaheads(e, e->d_chunks.get(), e->d_chunk_items.get(), e->n_resident > 0 ? e->res_grid : 0, e->d_items.get(), n_nonres,
                                   e->d_counters.get(), e->res.view(), e->pool.view(), e->d_stats.get(), st);
        if (rc != RAMP_OK) return rc;
        if (!capturing) {
            CUDA_TRY(cudaEventRecord(e->ev_b[e->ev_pending].get(), st));
            e->ev_pending++;
        }
    }
    launch_step_kernel(e, d_actions, fuse, d_stats_out, d_ncs_out);
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

int ramp_sync(ramp_engine_t* e) {
    if (!e) return set_error(RAMP_ERR_BAD_ARG, "null engine");
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    return resolve_events(e);
}

int ramp_step_host(ramp_engine_t* e, const ramp_action_t* actions, int32_t fuse, double* stats_out, int32_t* ncs_out) {
    if (!e || !actions) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    const int B = e->cfg.n_episodes;
    CUDA_TRY(cudaMemcpyAsync(e->d_actions.get(), actions, sizeof(ramp_action_t) * B, cudaMemcpyHostToDevice, e->stream.get()));
    int rc = ramp_step_device(e, e->d_actions.get(), fuse, stats_out ? e->d_step_stats.get() : nullptr, ncs_out ? e->d_n_cluster_steps.get() : nullptr);
    if (rc != RAMP_OK) return rc;
    if (stats_out)
        CUDA_TRY(cudaMemcpyAsync(stats_out, e->d_step_stats.get(), sizeof(double) * RAMP_STEP_STATS_LEN * B, cudaMemcpyDeviceToHost, e->stream.get()));
    if (ncs_out)
        CUDA_TRY(cudaMemcpyAsync(ncs_out, e->d_n_cluster_steps.get(), sizeof(int32_t) * B, cudaMemcpyDeviceToHost, e->stream.get()));
    return ramp_sync(e);
}

int ramp_check_status(ramp_engine_t* e, int32_t* ep_out, int32_t* st_out) {
    if (!e) return set_error(RAMP_ERR_BAD_ARG, "null engine");
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    Counters c{};
    CUDA_TRY(cudaMemcpy(&c, e->d_counters.get(), sizeof(Counters), cudaMemcpyDeviceToHost));
    if (c.err_episode == 0) { if (ep_out) *ep_out = -1; if (st_out) *st_out = 0; return RAMP_OK; }
    const int b = c.err_episode - 1;
    int32_t st = 0;
    CUDA_TRY(cudaMemcpy(&st, e->ep.ei + (size_t)EI_STATUS * e->cfg.n_episodes + b, sizeof(int32_t), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemset(&e->d_counters.get()->err_episode, 0, sizeof(int32_t)));
    if (ep_out) *ep_out = b;
    if (st_out) *st_out = st;
    const char* what = st == RAMP_ST_INFINITE_TICK ? "ERROR: Last tick was infinite, a bug has occurred somewhere."
                     : st == RAMP_ST_TRACE_OVERFLOW ? "lookahead needed more ticks than trace_cap (or the trace pool is full)"
                     : st == RAMP_ST_TABLE_FULL ? "running-job table or memo table is full"
                     : st == RAMP_ST_NO_QUEUED_JOB ? "an action was given for an episode whose job queue is empty"
                     : st == RAMP_ST_BAD_TEMPLATE ? "an action names a template id that was never registered"
                     : "simulation error";
    return set_error(RAMP_ERR_SIM, "episode %d: %s (status %d)", b, what, st);
}

int ramp_get_job_records(ramp_engine_t* e, ramp_job_record_t* out) {
    if (!e || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    CUDA_TRY(cudaMemcpy(out, e->ep.rec, sizeof(ramp_job_record_t) * (size_t)e->cfg.max_jobs * e->cfg.n_episodes, cudaMemcpyDeviceToHost));
    return RAMP_OK;
}

int ramp_episode_state_device(ramp_engine_t* e, double** d_out) {
    if (!e || !d_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    const int B = e->cfg.n_episodes;
    ramp_export_episode_state_kernel<<<(B + 127) / 128, 128, 0, e->stream.get()>>>(e->ep, e->d_ep_export.get());
    e->launches++;
    CUDA_TRY(cudaGetLastError());
    *d_out = e->d_ep_export.get();
    return RAMP_OK;
}

int ramp_export_episode_state_to(ramp_engine_t* e, double* d_dst) {
    if (!e || !d_dst) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    const int B = e->cfg.n_episodes;
    ramp_export_episode_state_kernel<<<(B + 127) / 128, 128, 0, e->stream.get()>>>(e->ep, d_dst);
    e->launches++;
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

int ramp_get_episode_state(ramp_engine_t* e, double* out) {
    double* d = nullptr;
    int rc = ramp_episode_state_device(e, &d);
    if (rc != RAMP_OK) return rc;
    CUDA_TRY(cudaMemcpyAsync(out, d, sizeof(double) * RAMP_EP_LEN * e->cfg.n_episodes, cudaMemcpyDeviceToHost, e->stream.get()));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    return RAMP_OK;
}

int ramp_get_memo_stats(ramp_engine_t* e, int64_t* lookups, int64_t* hits, int64_t* lookaheads) {
    if (!e) return set_error(RAMP_ERR_BAD_ARG, "null engine");
    // the counters and their copy at the last reset, in stream order: one synchronisation
    CUDA_TRY(cudaMemcpyAsync(e->h_stats.get(), e->d_stats.get(), 2 * sizeof(MemoStats), cudaMemcpyDeviceToHost, e->stream.get()));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    const MemoStats* s = e->h_stats.get();
    if (lookups) *lookups = (int64_t)(s[0].lookups - s[1].lookups);
    if (hits) *hits = (int64_t)(s[0].hits - s[1].hits);
    if (lookaheads) *lookaheads = (int64_t)(s[0].lookaheads - s[1].lookaheads);
    return RAMP_OK;
}

int ramp_get_memo_stats_ex(ramp_engine_t* e, int64_t out[4]) {
    if (!e || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    CUDA_TRY(cudaMemcpyAsync(e->h_stats.get(), e->d_stats.get(), 2 * sizeof(MemoStats), cudaMemcpyDeviceToHost, e->stream.get()));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    const MemoStats* s = e->h_stats.get();
    out[0] = (int64_t)(s[0].lookups - s[1].lookups);
    out[1] = (int64_t)(s[0].hits - s[1].hits);
    out[2] = (int64_t)(s[0].shared_hits - s[1].shared_hits);
    out[3] = (int64_t)(s[0].lookaheads - s[1].lookaheads);
    return RAMP_OK;
}

int ramp_get_last_lookahead(ramp_engine_t* e, int32_t episode, ramp_lookahead_result_t* res, int32_t* tn, double* tt, int32_t cap) {
    if (!e || !res) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (episode < 0 || episode >= e->cfg.n_episodes) return set_error(RAMP_ERR_BAD_ARG, "episode out of range");
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    int32_t slot = -1;
    CUDA_TRY(cudaMemcpy(&slot, e->ep.ei + (size_t)EI_LAST_SLOT * e->cfg.n_episodes + episode, sizeof(int32_t), cudaMemcpyDeviceToHost));
    if (slot < 0) return set_error(RAMP_ERR_BAD_ARG, "episode %d has not mounted a job yet", episode);
    int64_t off = -1;
    CUDA_TRY(cudaMemcpy(&res->jct, e->res.jct.get() + slot, sizeof(double), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(&res->comm, e->res.comm.get() + slot, sizeof(double), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(&res->comp, e->res.comp.get() + slot, sizeof(double), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(&res->n_ticks, e->res.n_ticks.get() + slot, sizeof(int32_t), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(&res->status, e->res.status.get() + slot, sizeof(int32_t), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(&off, e->res.trace_off.get() + slot, sizeof(int64_t), cudaMemcpyDeviceToHost));
    if (tn && tt && off >= 0) {
        const int32_t n = std::min(std::min(res->n_ticks, cap), e->cfg.trace_cap);
        CUDA_TRY(cudaMemcpy(tn, e->pool.n_active.get() + off, sizeof(int32_t) * n, cudaMemcpyDeviceToHost));
        CUDA_TRY(cudaMemcpy(tt, e->pool.tick.get() + off, sizeof(double) * n, cudaMemcpyDeviceToHost));
    }
    return RAMP_OK;
}

int ramp_debug_template_info(ramp_engine_t* e, int32_t template_id, int32_t out[7], double* hint_jct) {
    if (!e || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (template_id < 0 || template_id >= (int32_t)e->templates.size()) return set_error(RAMP_ERR_BAD_ARG, "template id %d is not registered", template_id);
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    const TemplateDev& d = e->templates[template_id].dev;
    TemplateHints h{};
    double hj = 0.0;
    CUDA_TRY(cudaMemcpy(&h, e->d_hints.get() + template_id, sizeof(TemplateHints), cudaMemcpyDeviceToHost));
    CUDA_TRY(cudaMemcpy(&hj, e->d_hint_jct.get() + template_id, sizeof(double), cudaMemcpyDeviceToHost));
    out[0] = d.size_class; out[1] = d.res_n_ops; out[2] = d.res_n_deps;
    out[3] = h.n_ticks; out[4] = h.max_o; out[5] = h.max_f; out[6] = h.max_nf;
    if (hint_jct) *hint_jct = hj;
    return RAMP_OK;
}

int ramp_run_lookaheads(ramp_engine_t* e, const int32_t* template_ids, int32_t n, ramp_lookahead_result_t* results,
                        int32_t* trace_n, double* trace_tick, int32_t trace_cap, float* kernel_ms_out) {
    if (!e || !template_ids || !results || n < 0) return set_error(RAMP_ERR_BAD_ARG, "bad argument");
    if (n == 0) return RAMP_OK;
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    for (int32_t k = 0; k < n; ++k)
        if (template_ids[k] < 0 || template_ids[k] >= (int32_t)e->templates.size())
            return set_error(RAMP_ERR_BAD_ARG, "template id %d at %d is not registered", template_ids[k], k);
    // the step's two work lists: non-resident (CTA kernel) and resident (thread kernel), each in item order
    std::vector<WorkItem> lists[2];
    std::vector<int32_t> per_template(e->templates.size(), 0);
    for (int32_t k = 0; k < n; ++k) {
        const int32_t t = template_ids[k];
        const bool resident = e->templates[t].dev.size_class == 2;
        lists[resident].push_back(WorkItem{t, k, -1, 0});
        if (resident) per_template[t]++;
    }
    const int n_nonres = (int)lists[0].size(), n_res = (int)lists[1].size();
    int n_chunks = 0;                   // what ramp_bucket_kernel will make of the resident list
    for (int32_t m : per_template) n_chunks += (m + 31) / 32;
    int rc = RAMP_OK;
    if (n_nonres > 0) { rc = ensure_scratch(e); if (rc != RAMP_OK) return rc; }
    if (n_res > 0) { rc = ensure_thread_scratch(e); if (rc != RAMP_OK) return rc; }
    cudaStream_t st = e->stream.get();
    if (n > e->sa_cap) {
        CUDA_TRY(cudaStreamSynchronize(st));
        e->sa_cap = 0;                  // until every buffer has the new size
        CUDA_TRY(alloc_each(n, e->sa_res, e->sa_items, e->sa_rank, e->sa_chunks));
        CUDA_TRY(e->sa_chunk_items.alloc((size_t)n * 32));
        e->sa_cap = n;
    }
    if (!e->sa_counters.get()) CUDA_TRY(e->sa_counters.alloc(1));
    std::vector<WorkItem> items;
    items.reserve(n);
    for (const auto& l : lists) items.insert(items.end(), l.begin(), l.end());
    WorkItem* const d_nonres = e->sa_items.get();
    WorkItem* const d_res = d_nonres + n_nonres;
    Counters c{}; c.n_work = n_nonres; c.n_work_res = n_res;
    CUDA_TRY(cudaMemcpyAsync(e->sa_items.get(), items.data(), sizeof(WorkItem) * n, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(e->sa_counters.get(), &c, sizeof(Counters), cudaMemcpyHostToDevice, st));
    if (n_res > 0) bucket_resident(e, d_res, e->sa_counters.get(), e->sa_chunk_items.get(), e->sa_chunks.get(), e->sa_rank.get(),
                                    e->d_tcount.get(), e->d_tbase.get(), st);
    // traces of standalone runs go to a private pool sized n x trace_cap when requested
    TraceArrays priv;
    const bool want_trace = trace_n && trace_tick && trace_cap > 0;
    if (want_trace) {
        // the kernels allocate n_ticks entries per lookahead; truncated on copy-out
        CUDA_TRY(priv.alloc((uint64_t)n * (uint64_t)e->cfg.trace_cap));
        CUDA_TRY(cudaMemsetAsync(priv.top.get(), 0, sizeof(unsigned long long), st));
    }
    TracePool pool = want_trace ? priv.view() : e->pool.view();
    if (!want_trace) pool.top = nullptr;
    cudaEvent_t ea = e->ev_a[MAX_EVENT_PAIRS - 1].get(), eb = e->ev_b[MAX_EVENT_PAIRS - 1].get();
    if (e->ev_pending >= MAX_EVENT_PAIRS - 1) { CUDA_TRY(cudaStreamSynchronize(st)); rc = resolve_events(e); if (rc) return rc; }
    CUDA_TRY(cudaEventRecord(ea, st));
    rc = launch_lookaheads(e, e->sa_chunks.get(), e->sa_chunk_items.get(), n_res > 0 ? std::min(e->res_grid, n_chunks) : 0, d_nonres, n_nonres,
                           e->sa_counters.get(), e->sa_res.view(), pool, nullptr, st);
    if (rc != RAMP_OK) return rc;
    CUDA_TRY(cudaEventRecord(eb, st));
    CUDA_TRY(cudaGetLastError());
    std::vector<double> jct(n), comm(n), comp(n);
    std::vector<int32_t> nt(n), stt(n);
    std::vector<int64_t> off(n);
    CUDA_TRY(cudaMemcpyAsync(jct.data(), e->sa_res.jct.get(), sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(comm.data(), e->sa_res.comm.get(), sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(comp.data(), e->sa_res.comp.get(), sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(nt.data(), e->sa_res.n_ticks.get(), sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(stt.data(), e->sa_res.status.get(), sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(off.data(), e->sa_res.trace_off.get(), sizeof(int64_t) * n, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (kernel_ms_out) CUDA_TRY(cudaEventElapsedTime(kernel_ms_out, ea, eb));
    for (int32_t k = 0; k < n; ++k) {
        results[k].jct = jct[k]; results[k].comm = comm[k]; results[k].comp = comp[k];
        results[k].n_ticks = nt[k]; results[k].status = stt[k];
    }
    if (want_trace) {
        for (int32_t k = 0; k < n; ++k) {
            if (off[k] < 0) continue;
            const int32_t m = std::min(std::min(nt[k], trace_cap), e->cfg.trace_cap);
            CUDA_TRY(cudaMemcpy(trace_n + (size_t)k * trace_cap, priv.n_active.get() + off[k], sizeof(int32_t) * m, cudaMemcpyDeviceToHost));
            CUDA_TRY(cudaMemcpy(trace_tick + (size_t)k * trace_cap, priv.tick.get() + off[k], sizeof(double) * m, cudaMemcpyDeviceToHost));
        }
    }
    return RAMP_OK;
}

int64_t ramp_launch_count(ramp_engine_t* e) { return e ? e->launches : 0; }

int ramp_debug_device_bytes(int64_t* device_bytes, int64_t* pinned_bytes) {
    if (device_bytes) *device_bytes = g_device_bytes.load();
    if (pinned_bytes) *pinned_bytes = g_pinned_bytes.load();
    return RAMP_OK;
}

int ramp_get_lookahead_kernel_time(ramp_engine_t* e, double* total_ms, int64_t* launches, int64_t* work_items,
                                   int64_t* alg_bytes, int32_t reset) {
    if (!e) return set_error(RAMP_ERR_BAD_ARG, "null engine");
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    int rc = resolve_events(e);
    if (rc) return rc;
    MemoStats s{};
    CUDA_TRY(cudaMemcpy(&s, e->d_stats.get(), sizeof(MemoStats), cudaMemcpyDeviceToHost));
    if (total_ms) *total_ms = e->la_ms_total;
    if (launches) *launches = e->la_launches;
    if (work_items) *work_items = (int64_t)(s.lookaheads - e->la_items_base);
    if (alg_bytes) *alg_bytes = (int64_t)(s.alg_bytes - e->la_bytes_base);
    if (reset) { e->la_ms_total = 0.0; e->la_ms_union = 0.0; e->la_launches = 0; e->la_items_base = s.lookaheads; e->la_bytes_base = s.alg_bytes; e->la_qbytes_base = s.quotient_bytes; }
    return RAMP_OK;
}


int ramp_get_lookahead_kernel_union(ramp_engine_t* e, double* union_ms) {
    if (!e || !union_ms) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    int rc = resolve_events(e);
    if (rc) return rc;
    *union_ms = e->la_ms_union;
    return RAMP_OK;
}

int ramp_get_memo_speculative_unused(ramp_engine_t* e, int64_t* unused) {
    if (!e || !unused) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    CUDA_TRY(cudaMemcpyAsync(e->h_stats.get(), e->d_stats.get(), 2 * sizeof(MemoStats), cudaMemcpyDeviceToHost, e->stream.get()));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    const MemoStats* s = e->h_stats.get();
    *unused = (int64_t)((s[0].lookaheads - s[1].lookaheads) - (s[0].ran - s[1].ran));
    return RAMP_OK;
}

int ramp_get_quotient_bytes(ramp_engine_t* e, int64_t* quotient_bytes) {
    if (!e || !quotient_bytes) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    MemoStats s{};
    CUDA_TRY(cudaMemcpy(&s, e->d_stats.get(), sizeof(MemoStats), cudaMemcpyDeviceToHost));
    *quotient_bytes = (int64_t)(s.quotient_bytes - e->la_qbytes_base);
    return RAMP_OK;
}


// ---- device-resident rollouts ---------------------------------------------------------------------------------------

int ramp_env_create(ramp_engine_t* e, const ramp_env_config_t* c) {
    if (!e || !c) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (e->has_env) return set_error(RAMP_ERR_BAD_ARG, "the engine already has an environment");
    const int B = e->cfg.n_episodes, J = c->jobs_per_episode, M = c->n_models, D = c->max_degree, G = c->n_geoms, nw = c->n_words;
    const int n_workers = c->shape[0] * c->shape[1] * c->shape[2];
    if (J != e->cfg.max_jobs) return set_error(RAMP_ERR_BAD_ARG, "jobs_per_episode %d != the engine's max_jobs %d", J, e->cfg.max_jobs);
    if (n_workers != e->cfg.n_cluster_workers || nw * 64 < n_workers || M < 1 || D < 1 || G < 1)
        return set_error(RAMP_ERR_BAD_ARG, "bad environment shape");
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    EnvDev& v = e->env;
    for (int k = 0; k < 3; ++k) e->env_shape[k] = c->shape[k];
    v.B = B; v.J = J; v.n_words = nw; v.n_models = M; v.max_degree = D; v.n_geoms = G; v.n_workers = n_workers;
    v.apply_mask = c->apply_action_mask; v.fail_reward = c->fail_reward; v.success_reward = c->success_reward;
    v.num_training_steps = (double)c->num_training_steps;
    v.machine_epsilon = c->machine_epsilon;
    const int n_cand = c->cand_ptr[D + 1];
    int rc;
    if ((rc = env_upload(e, &v.cand_ptr, c->cand_ptr, (size_t)D + 2))) return rc;
    if ((rc = env_upload(e, &v.cand_mask, c->cand_mask, (size_t)n_cand * nw))) return rc;
    if ((rc = env_upload(e, &v.cand_geom, c->cand_geom, (size_t)n_cand))) return rc;
    if ((rc = env_upload(e, &v.uniform, c->uniform, (size_t)M * (D + 1)))) return rc;
    if ((rc = env_upload(e, &v.shape_ok, c->shape_ok, (size_t)D + 1))) return rc;
    if ((rc = env_upload(e, &v.model_params, c->model_params, (size_t)M * 5))) return rc;
    if ((rc = env_upload(e, &v.jobs_params, c->jobs_params, (size_t)16))) return rc;
    std::vector<int32_t> minus1((size_t)M * (D + 1) * G, -1);
    if ((rc = env_upload(e, &v.tmpl_of, minus1.data(), minus1.size()))) return rc;
    if ((rc = env_upload<double>(e, &v.tmpl_mount, nullptr, (size_t)e->cfg.max_templates * 6))) return rc;
    if ((rc = env_upload(e, &v.model_of, nullptr, (size_t)B * J))) return rc;
    if ((rc = env_upload(e, &v.frac, nullptr, (size_t)B * J))) return rc;
    if ((rc = env_upload(e, &v.macc, nullptr, (size_t)B * J))) return rc;
    if ((rc = env_upload<unsigned long long>(e, &v.busy, nullptr, (size_t)B * nw))) return rc;
    if ((rc = env_upload<unsigned long long>(e, &v.job_mask, nullptr, (size_t)B * J * nw))) return rc;
    if ((rc = env_upload<unsigned long long>(e, &v.placed, nullptr, (size_t)B * nw))) return rc;
    if ((rc = env_upload<int32_t>(e, &v.tid, nullptr, (size_t)B))) return rc;
    if ((rc = env_upload<int32_t>(e, &v.decided_job, nullptr, (size_t)B))) return rc;
    if ((rc = env_upload<int32_t>(e, &v.n_decided, nullptr, (size_t)B))) return rc;
    if ((rc = env_upload<int32_t>(e, &v.job_tmpl, nullptr, (size_t)B * J))) return rc;
    if ((rc = env_upload<double>(e, &v.ret, nullptr, (size_t)B))) return rc;
    if ((rc = env_upload<int32_t>(e, &v.agent_kind, nullptr, (size_t)B))) return rc;
    if ((rc = env_upload<int32_t>(e, &v.agent_param, nullptr, (size_t)B))) return rc;
    if ((rc = env_upload<int32_t>(e, &v.actions, nullptr, (size_t)B))) return rc;
    if ((rc = env_upload<double>(e, &v.reward, nullptr, (size_t)B))) return rc;
    if ((rc = env_upload<uint8_t>(e, &v.done, nullptr, (size_t)B))) return rc;
    if ((rc = env_upload<int32_t>(e, &v.queued_model, nullptr, (size_t)B))) return rc;
    if ((rc = env_upload<float>(e, &v.obs_dyn, nullptr, (size_t)B * 11))) return rc;
    if ((rc = env_upload<uint8_t>(e, &v.action_mask, nullptr, (size_t)B * (D + 1)))) return rc;
    if ((rc = env_upload<int32_t>(e, &v.need_host, nullptr, (size_t)B))) return rc;
    if ((rc = env_upload<int32_t>(e, &v.n_need_host, nullptr, 1))) return rc;
    if ((rc = env_upload<int32_t>(e, &v.err, nullptr, 1))) return rc;
    CUDA_TRY(e->env_h_need.alloc(8));
    e->has_env = true;
    return RAMP_OK;
}

int ramp_env_set_template(ramp_engine_t* e, int32_t model, int32_t degree, int32_t geom, int32_t template_id, const double mount[6]) {
    if (!e || !e->has_env || !mount) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    const EnvDev& v = e->env;
    if (model < 0 || model >= v.n_models || degree < 0 || degree > v.max_degree || geom < 0 || geom >= v.n_geoms ||
        template_id < 0 || template_id >= (int32_t)e->templates.size())
        return set_error(RAMP_ERR_BAD_ARG, "bad template table entry (model %d degree %d geometry %d template %d)", model, degree, geom, template_id);
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaMemcpy(v.tmpl_of + ((size_t)model * (v.max_degree + 1) + degree) * v.n_geoms + geom, &template_id, sizeof(int32_t), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(v.tmpl_mount + (size_t)template_id * 6, mount, sizeof(double) * 6, cudaMemcpyHostToDevice));
    return RAMP_OK;
}

int ramp_env_set_placer_tables(ramp_engine_t* e, const ramp_env_placer_tables_t* t) {
    if (!e || !e->has_env || !t || !t->op_ptr || !t->topo || !t->par_ptr || !t->parents || !t->need || !t->splits || !t->cand_offset ||
        !t->cand_servers)
        return set_error(RAMP_ERR_BAD_ARG, "no environment or a null table");
    if (e->has_placer) return set_error(RAMP_ERR_BAD_ARG, "the environment already has its placer tables");
    const EnvDev& v = e->env;
    const int M = v.n_models, D = v.max_degree, N = t->n_ops_total, W = v.n_workers;
    int max_ops = 0;
    for (int m = 0; m < M; ++m) max_ops = std::max(max_ops, t->op_ptr[m + 1] - t->op_ptr[m]);
    if (t->op_ptr[0] != 0 || t->op_ptr[M] != N || N < 1) return set_error(RAMP_ERR_BAD_ARG, "op_ptr does not cover n_ops_total");
    PlaceDev p{};
    p.n_ops_total = N; p.capacity = t->memory_capacity;
    p.smem_mem_words = W + 8;
    p.smem_bytes_per_warp = (8 * p.smem_mem_words + 4 * max_ops + 7) / 8 * 8;
    if (p.smem_bytes_per_warp > RAMP_ENV_PLACE_SMEM_PER_WARP)
        return set_error(RAMP_ERR_BAD_ARG, "device placement needs %d bytes of shared memory per warp (%d servers, %d ops); the limit is %d",
                         p.smem_bytes_per_warp, W, max_ops, RAMP_ENV_PLACE_SMEM_PER_WARP);
    p.shape_r = e->env_shape[1]; p.shape_s = e->env_shape[2];
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    std::vector<int32_t> cand_ptr((size_t)D + 2);
    CUDA_TRY(cudaMemcpy(cand_ptr.data(), v.cand_ptr, sizeof(int32_t) * (D + 2), cudaMemcpyDeviceToHost));
    const int n_cand = cand_ptr[D + 1];
    int rc;
    if ((rc = env_upload(e, &p.op_ptr, t->op_ptr, (size_t)M + 1))) return rc;
    if ((rc = env_upload(e, &p.topo, t->topo, (size_t)N))) return rc;
    if ((rc = env_upload(e, &p.par_ptr, t->par_ptr, (size_t)N + 1))) return rc;
    if ((rc = env_upload(e, &p.parents, t->parents, (size_t)t->par_ptr[N]))) return rc;
    if ((rc = env_upload(e, &p.need, t->need, (size_t)N))) return rc;
    if ((rc = env_upload(e, &p.splits, t->splits, (size_t)(D + 1) * N))) return rc;
    if ((rc = env_upload(e, &p.cand_offset, t->cand_offset, (size_t)n_cand + 1))) return rc;
    if ((rc = env_upload(e, &p.cand_servers, t->cand_servers, (size_t)t->cand_offset[n_cand]))) return rc;
    if ((rc = env_upload<int32_t>(e, &p.host_list, nullptr, (size_t)v.B))) return rc;
    if ((rc = env_upload<int32_t>(e, &p.n_host, nullptr, 1))) return rc;
    const uint32_t cap = 64;
    e->place_keys.assign((size_t)cap * (v.n_words + 1), 0ull);
    e->place_tids.assign(cap, -1);
    e->place_count = 0;
    CUDA_TRY(e->place_table_keys.alloc(e->place_keys.size()));
    CUDA_TRY(e->place_table_tid.alloc(cap));
    CUDA_TRY(cudaMemcpy(e->place_table_keys.get(), e->place_keys.data(), sizeof(unsigned long long) * e->place_keys.size(), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(e->place_table_tid.get(), e->place_tids.data(), sizeof(int32_t) * cap, cudaMemcpyHostToDevice));
    p.table_keys = e->place_table_keys.get(); p.table_tid = e->place_table_tid.get(); p.table_mask = cap - 1;
    e->place = p;
    e->has_placer = true;
    return RAMP_OK;
}

// the slot of `key` ([n_words + 1]) in the host copy of the geometry table: its entry, or the empty slot that ends its probe
static uint32_t place_slot(const ramp_engine* e, const unsigned long long* key, uint32_t mask) {
    const int nw = e->env.n_words;
    unsigned long long h = 0ull;
    for (int w = 0; w <= nw; ++w) h = env_geom_hash_step(h, key[w]);
    for (uint32_t slot = (uint32_t)h & mask;; slot = (slot + 1) & mask) {
        const unsigned long long* k = e->place_keys.data() + (size_t)slot * (nw + 1);
        if (k[0] == 0ull || std::equal(k, k + nw + 1, key)) return slot;
    }
}

int ramp_env_set_geometry_template(ramp_engine_t* e, int32_t model, int32_t degree, const uint64_t* canonical_mask, int32_t template_id,
                                   const double mount[6]) {
    if (!e || !e->has_placer || !canonical_mask || !mount) return set_error(RAMP_ERR_BAD_ARG, "no placer tables or a null argument");
    const EnvDev& v = e->env;
    if (model < 0 || model >= v.n_models || degree < 1 || degree > v.max_degree || template_id < 0 || template_id >= (int32_t)e->templates.size())
        return set_error(RAMP_ERR_BAD_ARG, "bad geometry table entry (model %d degree %d template %d)", model, degree, template_id);
    const int nw = v.n_words;
    std::vector<unsigned long long> key((size_t)nw + 1);
    key[0] = ((unsigned long long)(model + 1) << 32) | (unsigned long long)degree;
    for (int w = 0; w < nw; ++w) key[1 + w] = canonical_mask[w];
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    cudaStream_t st = e->stream.get();
    uint32_t cap = (uint32_t)e->place_tids.size();
    uint32_t slot = place_slot(e, key.data(), cap - 1);
    const bool fresh = e->place_keys[(size_t)slot * (nw + 1)] == 0ull;
    if (fresh && 2 * (e->place_count + 1) > cap) {
        // at most half full: rehash the host copy into twice the slots and upload it whole
        std::vector<unsigned long long> old_keys;
        std::vector<int32_t> old_tids;
        old_keys.swap(e->place_keys); old_tids.swap(e->place_tids);
        cap *= 2;
        e->place_keys.assign((size_t)cap * (nw + 1), 0ull);
        e->place_tids.assign(cap, -1);
        for (size_t o = 0; o < old_tids.size(); ++o) {
            const unsigned long long* k = old_keys.data() + o * (nw + 1);
            if (k[0] == 0ull) continue;
            const uint32_t to = place_slot(e, k, cap - 1);
            std::copy(k, k + nw + 1, e->place_keys.begin() + (size_t)to * (nw + 1));
            e->place_tids[to] = old_tids[o];
        }
        DeviceArray<unsigned long long> keys;
        DeviceArray<int32_t> tids;
        CUDA_TRY(keys.alloc(e->place_keys.size()));
        CUDA_TRY(tids.alloc(cap));
        CUDA_TRY(cudaMemcpyAsync(keys.get(), e->place_keys.data(), sizeof(unsigned long long) * e->place_keys.size(), cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(tids.get(), e->place_tids.data(), sizeof(int32_t) * cap, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        e->place_table_keys = std::move(keys);            // frees the old table: no kernel queued on the stream reads it any more
        e->place_table_tid = std::move(tids);
        e->place.table_keys = e->place_table_keys.get(); e->place.table_tid = e->place_table_tid.get(); e->place.table_mask = cap - 1;
        slot = place_slot(e, key.data(), cap - 1);
    }
    if (fresh) e->place_count++;
    std::copy(key.begin(), key.end(), e->place_keys.begin() + (size_t)slot * (nw + 1));
    e->place_tids[slot] = template_id;
    // on the engine stream, behind every kernel queued so far (pageable sources: the copies are staged before the calls return)
    CUDA_TRY(cudaMemcpyAsync(v.tmpl_mount + (size_t)template_id * 6, mount, sizeof(double) * 6, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(e->place_table_tid.get() + slot, &e->place_tids[slot], sizeof(int32_t), cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(e->place_table_keys.get() + (size_t)slot * (nw + 1), key.data(), sizeof(unsigned long long) * (nw + 1),
                             cudaMemcpyHostToDevice, st));
    return RAMP_OK;
}

int ramp_env_reset(ramp_engine_t* e, const int32_t* model_of, const double* frac, const double* macc, const ramp_arrival_t* arrivals) {
    if (!e || !e->has_env || !model_of || !frac || !macc || !arrivals) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    EnvDev& v = e->env;
    const size_t n = (size_t)v.B * v.J;
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaMemcpyAsync((void*)v.model_of, model_of, sizeof(int32_t) * n, cudaMemcpyHostToDevice, e->stream.get()));
    CUDA_TRY(cudaMemcpyAsync((void*)v.frac, frac, sizeof(double) * n, cudaMemcpyHostToDevice, e->stream.get()));
    CUDA_TRY(cudaMemcpyAsync((void*)v.macc, macc, sizeof(double) * n, cudaMemcpyHostToDevice, e->stream.get()));
    CUDA_TRY(cudaMemsetAsync(v.job_mask, 0, sizeof(unsigned long long) * n * v.n_words, e->stream.get()));
    CUDA_TRY(cudaMemsetAsync(v.done, 0, (size_t)v.B, e->stream.get()));
    CUDA_TRY(cudaMemsetAsync(v.n_decided, 0, sizeof(int32_t) * (size_t)v.B, e->stream.get()));
    CUDA_TRY(cudaMemsetAsync(v.job_tmpl, 0xFF, sizeof(int32_t) * n, e->stream.get()));          // -1
    CUDA_TRY(cudaMemsetAsync(v.ret, 0, sizeof(double) * (size_t)v.B, e->stream.get()));
    CUDA_TRY(cudaMemsetAsync(v.err, 0, sizeof(int32_t), e->stream.get()));
    if (e->env_range_err.get()) {
        CUDA_TRY(cudaMemsetAsync(e->env_range_err.get(), 0xFF, sizeof(unsigned long long), e->stream.get()));
        CUDA_TRY(cudaMemsetAsync(e->env_ingest_seq.get(), 0, sizeof(uint32_t), e->stream.get()));
        e->env_range_armed = false;
    }
    int rc = ramp_reset(e, arrivals, v.J);
    if (rc != RAMP_OK) return rc;
    ramp_env_update_kernel<<<(v.B + 127) / 128, 128, 0, e->stream.get()>>>(v, e->ep, nullptr, 1);
    e->launches++;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    return RAMP_OK;
}

int ramp_env_buffers(ramp_engine_t* e, ramp_env_buffers_t* out) {
    if (!e || !e->has_env || !out) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    const EnvDev& v = e->env;
    out->actions = v.actions; out->reward = v.reward; out->done = v.done; out->queued_model = v.queued_model;
    out->obs_dynamic = v.obs_dyn; out->action_mask = v.action_mask; out->busy = (uint64_t*)v.busy; out->template_id = v.tid;
    out->n_episodes = v.B; out->n_actions = v.max_degree + 1; out->n_models = v.n_models;
    return RAMP_OK;
}

int ramp_env_host_mirror(ramp_engine_t* e, ramp_env_buffers_t* out) {
    if (!e || !e->has_env || !out) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    const EnvDev& v = e->env;
    const size_t B = (size_t)v.B, A = (size_t)v.max_degree + 1;
    const size_t o_reward = 0, o_obs = o_reward + 8 * B, o_act = o_obs + 44 * B, o_qm = o_act + 4 * B, o_done = o_qm + 4 * B, o_mask = o_done + B;
    if (!e->env_h_mirror.get()) {
        CUDA_TRY(cudaSetDevice(e->cfg.device));
        CUDA_TRY(e->env_h_mirror.alloc(o_mask + B * A + 64));
        memset(e->env_h_mirror.get(), 0, o_mask + B * A + 64);
    }
    unsigned char* m = e->env_h_mirror.get();
    memset(out, 0, sizeof(*out));
    out->reward = (double*)(m + o_reward); out->obs_dynamic = (float*)(m + o_obs); out->actions = (int32_t*)(m + o_act);
    out->queued_model = (int32_t*)(m + o_qm); out->done = m + o_done; out->action_mask = m + o_mask;
    out->n_episodes = v.B; out->n_actions = v.max_degree + 1; out->n_models = v.n_models;
    return RAMP_OK;
}

int ramp_env_decide(ramp_engine_t* e, const int32_t* actions, int32_t* n_need_host_out, int32_t* need_host_out) {
    if (!e || !e->has_env) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    EnvDev& v = e->env;
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    cudaStream_t st = e->stream.get();
    if (n_need_host_out || actions) {
        bool capturing = false;
        int rc = capture_status(st, &capturing);
        if (rc != RAMP_OK) return rc;
        if (capturing)
            return set_error(RAMP_ERR_BAD_ARG, "CUDA-graph capture refused: a captured decision can neither take host actions nor "
                             "hand episodes to the host's placer");
    }
    if (actions) CUDA_TRY(cudaMemcpyAsync(v.actions, actions, sizeof(int32_t) * v.B, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(v.n_need_host, 0, sizeof(int32_t), st));
    ramp_env_decide_kernel<<<(v.B + 127) / 128, 128, 0, st>>>(v, e->ep, e->d_actions.get());
    e->launches++;
    CUDA_TRY(cudaGetLastError());
    if (e->has_placer) {
        // the decide kernel's list length stays on the device: the grid covers every episode and each warp reads the length
        const PlaceDev& p = e->place;
        CUDA_TRY(cudaMemsetAsync(p.n_host, 0, sizeof(int32_t), st));
        const int grid = std::max(1, std::min((v.B + ENV_PLACE_WARPS - 1) / ENV_PLACE_WARPS, e->sm_count * 4));
        ramp_env_place_kernel<<<grid, ENV_PLACE_WARPS * 32, (size_t)ENV_PLACE_WARPS * p.smem_bytes_per_warp, st>>>(v, p, e->d_actions.get());
        e->launches++;
        CUDA_TRY(cudaGetLastError());
    }
    const int32_t* host_count = e->has_placer ? e->place.n_host : v.n_need_host;
    const int32_t* host_list = e->has_placer ? e->place.host_list : v.need_host;
    if (n_need_host_out) {
        CUDA_TRY(cudaMemcpyAsync(e->env_h_need.get(), host_count, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(e->env_h_need.get() + 1, v.err, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        const bool range = e->env_range_armed || e->env_captured;
        if (range) { int rc = env_range_fetch(e); if (rc != RAMP_OK) return rc; }
        CUDA_TRY(cudaStreamSynchronize(st));
        if (range) { int rc = env_range_raise(e); if (rc != RAMP_OK) return rc; }
        if (e->env_h_need.get()[1] != 0) {
            CUDA_TRY(cudaMemset(v.err, 0, sizeof(int32_t)));
            return set_error(RAMP_ERR_BAD_ARG, "episode %d: the action is invalid given its action mask (RJPE:314-319)", e->env_h_need.get()[1] - 1);
        }
        *n_need_host_out = e->env_h_need.get()[0];
        if (need_host_out && e->env_h_need.get()[0] > 0)
            CUDA_TRY(cudaMemcpy(need_host_out, host_list, sizeof(int32_t) * e->env_h_need.get()[0], cudaMemcpyDeviceToHost));
    } else {
        e->env_unchecked_decide = true;      // looked at by the next ramp_env_read
    }
    return RAMP_OK;
}

int ramp_env_patch(ramp_engine_t* e, int32_t episode, int32_t template_id, const uint64_t* server_mask, const double mount[6]) {
    if (!e || !e->has_env || !server_mask || !mount) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    EnvDev& v = e->env;
    if (episode < 0 || episode >= v.B || template_id >= (int32_t)e->templates.size()) return set_error(RAMP_ERR_BAD_ARG, "bad patch");
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    int32_t q = -1;
    CUDA_TRY(cudaMemcpy(&q, v.decided_job + episode, sizeof(int32_t), cudaMemcpyDeviceToHost));
    ramp_action_t row{};
    row.template_id = template_id;
    if (template_id >= 0 && q >= 0) {
        double fr = 0.0, ov = 0.0;
        CUDA_TRY(cudaMemcpy(&fr, v.frac + (size_t)episode * v.J + q, sizeof(double), cudaMemcpyDeviceToHost));
        CUDA_TRY(cudaMemcpy(&ov, v.macc + (size_t)episode * v.J + q, sizeof(double), cudaMemcpyDeviceToHost));
        row.max_acceptable_jct = std::isnan(ov) ? fr * mount[0] : ov;
        row.part_op_mem = mount[1]; row.part_dep_size = mount[2]; row.flow_size = mount[3];
        row.n_mounted_workers = (int32_t)mount[4]; row.n_mounted_channels = (int32_t)mount[5];
    } else {
        row.template_id = -1;
    }
    CUDA_TRY(cudaMemcpy(e->d_actions.get() + episode, &row, sizeof(row), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(v.tid + episode, &row.template_id, sizeof(int32_t), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMemcpy(v.placed + (size_t)episode * v.n_words, server_mask, sizeof(uint64_t) * v.n_words, cudaMemcpyHostToDevice));
    return RAMP_OK;
}

int ramp_env_advance(ramp_engine_t* e) {
    if (!e || !e->has_env) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    EnvDev& v = e->env;
    int rc = ramp_step_device(e, e->d_actions.get(), 1, e->d_step_stats.get(), e->d_n_cluster_steps.get());
    if (rc != RAMP_OK) return rc;
    ramp_env_update_kernel<<<(v.B + 127) / 128, 128, 0, e->stream.get()>>>(v, e->ep, e->d_n_cluster_steps.get(), 0);
    e->launches++;
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

int ramp_env_read(ramp_engine_t* e, double* reward, uint8_t* done, int32_t* queued_model, float* obs_dynamic, uint8_t* action_mask) {
    if (!e || !e->has_env) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    const EnvDev& v = e->env;
    cudaStream_t st = e->stream.get();
    if (reward) CUDA_TRY(cudaMemcpyAsync(reward, v.reward, sizeof(double) * v.B, cudaMemcpyDeviceToHost, st));
    if (done) CUDA_TRY(cudaMemcpyAsync(done, v.done, (size_t)v.B, cudaMemcpyDeviceToHost, st));
    if (queued_model) CUDA_TRY(cudaMemcpyAsync(queued_model, v.queued_model, sizeof(int32_t) * v.B, cudaMemcpyDeviceToHost, st));
    if (obs_dynamic) CUDA_TRY(cudaMemcpyAsync(obs_dynamic, v.obs_dyn, sizeof(float) * 11 * v.B, cudaMemcpyDeviceToHost, st));
    if (action_mask) CUDA_TRY(cudaMemcpyAsync(action_mask, v.action_mask, (size_t)v.B * (v.max_degree + 1), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(e->env_h_need.get() + 4, &e->d_counters.get()->err_episode, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    if (e->env_unchecked_decide || e->env_captured) {
        // decisions taken without the host looking (a device-resident policy, a replayed CUDA graph): an invalid action under
        // apply_action_mask is sticky in `err`; episodes the tables could not decide were left unplaced, which only the LAST
        // decide's count can show
        CUDA_TRY(cudaMemcpyAsync(e->env_h_need.get() + 2, e->has_placer ? e->place.n_host : v.n_need_host, sizeof(int32_t),
                                 cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(e->env_h_need.get() + 3, v.err, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
        const bool range = e->env_range_armed || e->env_captured;
        int rc = range ? env_range_fetch(e) : RAMP_OK;
        if (rc != RAMP_OK) return rc;
        rc = ramp_sync(e);
        if (rc != RAMP_OK) return rc;
        e->env_unchecked_decide = false;
        if (range && (rc = env_range_raise(e)) != RAMP_OK) return rc;      // RJPE:314-316 before 317-319
        if (e->env_h_need.get()[3] != 0) {
            CUDA_TRY(cudaMemset(v.err, 0, sizeof(int32_t)));
            return set_error(RAMP_ERR_BAD_ARG, "episode %d: the action is invalid given its action mask (RJPE:314-319)", e->env_h_need.get()[3] - 1);
        }
        if (e->env_h_need.get()[2] != 0)
            return set_error(RAMP_ERR_BAD_ARG, "%d episodes needed the host's placer but ramp_env_decide was called without need_host_out", e->env_h_need.get()[2]);
        return e->env_h_need.get()[4] != 0 ? ramp_check_status(e, nullptr, nullptr) : RAMP_OK;
    }
    {
        const bool range = e->env_range_armed || e->env_captured;
        int rc = range ? env_range_fetch(e) : RAMP_OK;
        if (rc != RAMP_OK) return rc;
        rc = ramp_sync(e);
        if (rc != RAMP_OK) return rc;
        if (range && (rc = env_range_raise(e)) != RAMP_OK) return rc;
    }
    return e->env_h_need.get()[4] != 0 ? ramp_check_status(e, nullptr, nullptr) : RAMP_OK;
}

int ramp_env_set_graph_static(ramp_engine_t* e, const float* graph_static) {
    if (!e || !e->has_env || !graph_static) return set_error(RAMP_ERR_BAD_ARG, "no environment or no statistics");
    const size_t n = (size_t)e->env.n_models * ENV_GF_STATIC;
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));      // no export queued behind the engine stream still reads the old table
    if (!e->env_graph_static.get()) CUDA_TRY(e->env_graph_static.alloc(n));
    CUDA_TRY(cudaMemcpy(e->env_graph_static.get(), graph_static, sizeof(float) * n, cudaMemcpyHostToDevice));
    return RAMP_OK;
}

// RJPE:300-322 (the action, range-checked as RJPE:314-316 does) from caller-owned device memory, on the caller's stream
int ramp_env_ingest(ramp_engine_t* e, const void* actions, int32_t dtype, void* stream) {
    if (!e || !e->has_env) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    if (!actions) return set_error(RAMP_ERR_BAD_ARG, "null actions");
    if (dtype != RAMP_ACTIONS_INT32 && dtype != RAMP_ACTIONS_INT64)
        return set_error(RAMP_ERR_BAD_ARG, "actions dtype %d is neither RAMP_ACTIONS_INT32 nor RAMP_ACTIONS_INT64", dtype);
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    EnvDev& v = e->env;
    cudaStream_t cs = (cudaStream_t)stream, st = e->stream.get();
    bool capturing = false;
    int rc = capture_status(cs, &capturing);
    if (rc != RAMP_OK) return rc;
    if (capturing) {
        // the step's first call: every refusal of a captured step is decided here, before anything is enqueued
        if (!e->env_ev_to_engine)
            return set_error(RAMP_ERR_BAD_ARG, "CUDA-graph capture refused: no eager step has run yet to make the environment's i/o buffers");
        if ((rc = capture_refusal(e)) != RAMP_OK) return rc;
    } else {
        if ((rc = env_io_ready(e)) != RAMP_OK) return rc;
        // the last ramp_env_advance wrote `done` and read `actions` (its env-step record), both on the engine stream.  A capture
        // does not wait here: the graph's replays queue behind the caller's stream, which every eager call leaves behind the engine
        if ((rc = env_fence(e->env_ev_to_caller.get(), st, cs)) != RAMP_OK) return rc;
    }
    EnvIngestArgs a{};
    a.actions = actions; a.is64 = dtype == RAMP_ACTIONS_INT64; a.B = v.B; a.max_degree = v.max_degree; a.seq = e->env_ingest_seq.get();
    a.done = v.done; a.out = v.actions; a.range_err = e->env_range_err.get(); a.range_val = e->env_range_val.get();
    ramp_env_ingest_kernel<<<(v.B + 127) / 128, 128, 0, cs>>>(a);
    e->launches++;
    CUDA_TRY(cudaGetLastError());
    e->env_range_armed = true;
    // ramp_env_decide reads what the kernel wrote; under capture this forks the engine stream into the caller's capture, and
    // ramp_env_export joins it back
    return env_fence(e->env_ev_to_engine.get(), cs, st);
}

int ramp_env_join(ramp_engine_t* e, void* stream) {
    if (!e || !e->has_env) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    cudaStream_t cs = (cudaStream_t)stream;
    bool capturing = false;
    int rc = capture_status(cs, &capturing);
    if (rc != RAMP_OK) return rc;
    if (capturing) return set_error(RAMP_ERR_BAD_ARG, "ramp_env_join: the stream is capturing a CUDA graph; join after the replay");
    if ((rc = env_io_ready(e)) != RAMP_OK) return rc;
    return env_fence(e->env_ev_to_engine.get(), cs, e->stream.get());
}

// RampJobPartitioningObservation (ramp_job_partitioning_observation.py:275, observation.py:80-131, 358-498), reward and done of the
// last ramp_env_advance into caller-owned device memory, on the caller's stream
int ramp_env_export(ramp_engine_t* e, void* stream, const ramp_env_export_t* out) {
    if (!e || !e->has_env || !out) return set_error(RAMP_ERR_BAD_ARG, "no environment or no outputs");
    if (out->graph_features && !e->env_graph_static.get())
        return set_error(RAMP_ERR_BAD_ARG, "graph_features needs the per-graph statistics: call ramp_env_set_graph_static first");
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    const EnvDev& v = e->env;
    cudaStream_t cs = (cudaStream_t)stream, st = e->stream.get();
    bool capturing = false;
    int rc = capture_status(cs, &capturing);
    if (rc != RAMP_OK) return rc;
    if (capturing && !e->env_ev_to_engine)
        return set_error(RAMP_ERR_BAD_ARG, "CUDA-graph capture refused: no eager step has run yet to make the environment's i/o buffers");
    if (!capturing && (rc = env_io_ready(e)) != RAMP_OK) return rc;
    // ramp_env_update_kernel's outputs; under capture this joins the engine stream back into the caller's capture
    if ((rc = env_fence(e->env_ev_to_caller.get(), st, cs)) != RAMP_OK) return rc;
    EnvExportArgs a{};
    a.B = v.B; a.A = v.max_degree + 1; a.n_models = v.n_models;
    a.queued_model = v.queued_model; a.obs_dyn = v.obs_dyn; a.mask = v.action_mask; a.reward = v.reward; a.done = v.done;
    a.graph_static = e->env_graph_static.get();
    a.model = reinterpret_cast<long long*>(out->model); a.graph_features = out->graph_features; a.action_mask = out->action_mask;
    a.reward_out = out->reward; a.done_out = out->done;
    const long long n = (long long)v.B * (ENV_GF_BASE + a.A);
    ramp_env_export_kernel<<<(unsigned)((n + 255) / 256), 256, 0, cs>>>(a);
    e->launches++;
    CUDA_TRY(cudaGetLastError());
    if (capturing) {
        // no fork is left open: the next captured step's ingest orders the engine stream again, and after a replay the engine
        // stream's next work waits for the caller's stream through ramp_env_join or the next ingest
        e->env_captured = true;
        return RAMP_OK;
    }
    return env_fence(e->env_ev_to_engine.get(), cs, st);       // the next step's kernels overwrite what the kernel reads
}


int ramp_enable_tick_lists(ramp_engine_t* e, int32_t cap) {
    if (!e || cap < 1) return set_error(RAMP_ERR_BAD_ARG, "ramp_enable_tick_lists: cap must be >= 1");
    if (e->env_captured)
        return set_error(RAMP_ERR_BAD_ARG, "ramp_enable_tick_lists: a step was captured into a CUDA graph, whose step kernels keep the "
                         "lists' addresses");
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    e->ep.tick_util = nullptr; e->ep.tick_util_n = nullptr;     // no lists until both arrays are there
    const size_t B = (size_t)e->cfg.n_episodes;
    CUDA_TRY(e->tick_util.alloc(B * (size_t)cap * 2));
    CUDA_TRY(e->tick_util_n.alloc(B));
    CUDA_TRY(cudaMemset(e->tick_util_n.get(), 0, sizeof(int32_t) * B));
    e->ep.tick_util = e->tick_util.get(); e->ep.tick_util_n = e->tick_util_n.get(); e->ep.tick_util_cap = cap;
    return RAMP_OK;
}

int ramp_get_tick_lists(ramp_engine_t* e, int32_t episode, double* mounted_out, double* cluster_out, int32_t cap, int32_t* n_out) {
    if (!e || !n_out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (!e->ep.tick_util) return set_error(RAMP_ERR_BAD_ARG, "per-tick lists are not recorded (ramp_enable_tick_lists)");
    if (episode < 0 || episode >= e->cfg.n_episodes) return set_error(RAMP_ERR_BAD_ARG, "bad episode %d", episode);
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    int32_t n = 0;
    CUDA_TRY(cudaMemcpy(&n, e->ep.tick_util_n + episode, sizeof(int32_t), cudaMemcpyDeviceToHost));
    *n_out = n;
    if (n > e->ep.tick_util_cap)
        return set_error(RAMP_ERR_CAPACITY, "episode %d: the step had %d outer-loop iterations, the per-tick lists hold %d", episode, n, e->ep.tick_util_cap);
    const int m = std::min(n, cap);
    if (m > 0 && mounted_out && cluster_out) {
        std::vector<double> rows((size_t)m * 2);
        CUDA_TRY(cudaMemcpy(rows.data(), e->ep.tick_util + (size_t)episode * e->ep.tick_util_cap * 2, sizeof(double) * rows.size(), cudaMemcpyDeviceToHost));
        for (int k = 0; k < m; ++k) { mounted_out[k] = rows[2 * k]; cluster_out[k] = rows[2 * k + 1]; }
    }
    return RAMP_OK;
}

int ramp_get_last_step_stats(ramp_engine_t* e, double* stats_out, int32_t* n_cluster_steps_out) {
    if (!e) return set_error(RAMP_ERR_BAD_ARG, "null engine");
    const int B = e->cfg.n_episodes;
    if (stats_out) CUDA_TRY(cudaMemcpyAsync(stats_out, e->d_step_stats.get(), sizeof(double) * RAMP_STEP_STATS_LEN * B, cudaMemcpyDeviceToHost, e->stream.get()));
    if (n_cluster_steps_out) CUDA_TRY(cudaMemcpyAsync(n_cluster_steps_out, e->d_n_cluster_steps.get(), sizeof(int32_t) * B, cudaMemcpyDeviceToHost, e->stream.get()));
    return ramp_sync(e);
}


int ramp_enable_env_step_stats(ramp_engine_t* e) {
    if (!e) return set_error(RAMP_ERR_BAD_ARG, "null engine");
    if (e->ep.es) return RAMP_OK;
    const size_t B = (size_t)e->cfg.n_episodes;
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));
    CUDA_TRY(e->ep_es.alloc((size_t)ES_STRIDE * B));
    CUDA_TRY(cudaMemset(e->ep_es.get(), 0, sizeof(double) * ES_STRIDE * B));
    e->ep.es = e->ep_es.get();
    return RAMP_OK;
}

// eval_loop.py:50-100: the rows the step kernel closed, the first RAMP_ENV_STEP_STATS_LEN of every episode's ES_STRIDE
int ramp_get_env_step_stats(ramp_engine_t* e, double* out) {
    if (!e || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    if (!e->ep.es) return set_error(RAMP_ERR_BAD_ARG, "env-step statistics are not kept (ramp_enable_env_step_stats)");
    const size_t B = (size_t)e->cfg.n_episodes, K = RAMP_ENV_STEP_STATS_LEN;
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaMemcpy2DAsync(out, sizeof(double) * K, e->ep.es, sizeof(double) * ES_STRIDE, sizeof(double) * K, B,
                               cudaMemcpyDeviceToHost, e->stream.get()));
    return ramp_sync(e);
}

// eval_loop.py:44-100: results['step_stats'] of every episode, one row per env-step, written by ramp_env_update_kernel
int ramp_env_steplog_begin(ramp_engine_t* e, int32_t horizon) {
    if (!e || !e->has_env) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    if (horizon < 0) return set_error(RAMP_ERR_BAD_ARG, "horizon %d < 0", horizon);
    if (horizon > 0 && !e->ep.es) return set_error(RAMP_ERR_BAD_ARG, "env-step statistics are not kept (ramp_enable_env_step_stats)");
    EnvDev& v = e->env;
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaStreamSynchronize(e->stream.get()));      // no queued ramp_env_advance still writes the old record
    if (e->env_captured && horizon != v.log_horizon)
        return set_error(RAMP_ERR_BAD_ARG, "the env-step record of horizon %d is written by captured CUDA-graph steps; it can only be "
                         "cleared (horizon %d), not replaced by one of horizon %d", v.log_horizon, v.log_horizon, horizon);
    if (e->env_captured) {                                 // the same buffers, cleared: a graph's kernels keep their addresses
        const size_t n = (size_t)horizon * v.B;
        if (n) {
            CUDA_TRY(cudaMemset(v.log_stats, 0, sizeof(double) * n * RAMP_ENV_STEP_STATS_LEN));
            CUDA_TRY(cudaMemset(v.log_rewards, 0, sizeof(double) * n));
            CUDA_TRY(cudaMemset(v.log_actions, 0, sizeof(int32_t) * n));
        }
        return RAMP_OK;
    }
    v.log_horizon = 0; v.log_stats = nullptr; v.log_actions = nullptr; v.log_rewards = nullptr;
    e->steplog_stats = {}; e->steplog_actions = {}; e->steplog_rewards = {};
    if (horizon == 0) return RAMP_OK;
    const size_t n = (size_t)horizon * v.B;
    CUDA_TRY(e->steplog_stats.alloc(n * RAMP_ENV_STEP_STATS_LEN));
    CUDA_TRY(alloc_each(n, e->steplog_rewards));
    CUDA_TRY(alloc_each(n, e->steplog_actions));
    CUDA_TRY(cudaMemsetAsync(e->steplog_stats.get(), 0, sizeof(double) * n * RAMP_ENV_STEP_STATS_LEN, e->stream.get()));
    CUDA_TRY(cudaMemsetAsync(e->steplog_rewards.get(), 0, sizeof(double) * n, e->stream.get()));
    CUDA_TRY(cudaMemsetAsync(e->steplog_actions.get(), 0, sizeof(int32_t) * n, e->stream.get()));
    v.log_stats = e->steplog_stats.get(); v.log_actions = e->steplog_actions.get(); v.log_rewards = e->steplog_rewards.get();
    v.log_horizon = horizon;
    return RAMP_OK;
}

int ramp_env_steplog_read(ramp_engine_t* e, int32_t horizon, double* stats_out, int32_t* actions_out, double* rewards_out,
                          int32_t* n_steps_out) {
    if (!e || !e->has_env) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    const EnvDev& v = e->env;
    if (v.log_horizon <= 0) return set_error(RAMP_ERR_BAD_ARG, "no env-step record: call ramp_env_steplog_begin first");
    if (horizon != v.log_horizon) return set_error(RAMP_ERR_BAD_ARG, "horizon %d != the record's %d", horizon, v.log_horizon);
    const size_t n = (size_t)horizon * v.B;
    cudaStream_t st = e->stream.get();
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    if (stats_out) CUDA_TRY(cudaMemcpyAsync(stats_out, v.log_stats, sizeof(double) * n * RAMP_ENV_STEP_STATS_LEN, cudaMemcpyDeviceToHost, st));
    if (actions_out) CUDA_TRY(cudaMemcpyAsync(actions_out, v.log_actions, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    if (rewards_out) CUDA_TRY(cudaMemcpyAsync(rewards_out, v.log_rewards, sizeof(double) * n, cudaMemcpyDeviceToHost, st));
    if (n_steps_out) CUDA_TRY(cudaMemcpyAsync(n_steps_out, v.n_decided, sizeof(int32_t) * v.B, cudaMemcpyDeviceToHost, st));
    return ramp_sync(e);
}

int ramp_env_read_state(ramp_engine_t* e, uint64_t* busy_out, int32_t* actions_out, int32_t* n_decided_out) {
    if (!e || !e->has_env) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    const EnvDev& v = e->env;
    if (busy_out) CUDA_TRY(cudaMemcpyAsync(busy_out, v.busy, sizeof(uint64_t) * (size_t)v.B * v.n_words, cudaMemcpyDeviceToHost, e->stream.get()));
    if (actions_out) CUDA_TRY(cudaMemcpyAsync(actions_out, v.actions, sizeof(int32_t) * v.B, cudaMemcpyDeviceToHost, e->stream.get()));
    if (n_decided_out) CUDA_TRY(cudaMemcpyAsync(n_decided_out, v.n_decided, sizeof(int32_t) * v.B, cudaMemcpyDeviceToHost, e->stream.get()));
    return ramp_sync(e);
}

int ramp_env_read_episode(ramp_engine_t* e, int32_t* job_template_out, double* return_out) {
    if (!e || !e->has_env) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    const EnvDev& v = e->env;
    if (job_template_out)
        CUDA_TRY(cudaMemcpyAsync(job_template_out, v.job_tmpl, sizeof(int32_t) * (size_t)v.B * v.J, cudaMemcpyDeviceToHost, e->stream.get()));
    if (return_out) CUDA_TRY(cudaMemcpyAsync(return_out, v.ret, sizeof(double) * v.B, cudaMemcpyDeviceToHost, e->stream.get()));
    return ramp_sync(e);
}

int ramp_get_episode_stats(ramp_engine_t* e, double* out) {
    if (!e || !out) return set_error(RAMP_ERR_BAD_ARG, "null argument");
    const int B = e->cfg.n_episodes;
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    ramp_episode_stats_kernel<<<(B + 127) / 128, 128, 0, e->stream.get()>>>(e->ep, e->d_es_export.get());
    e->launches++;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(out, e->d_es_export.get(), sizeof(double) * RAMP_ES_LEN * B, cudaMemcpyDeviceToHost, e->stream.get()));
    return ramp_sync(e);
}

int ramp_env_set_agents(ramp_engine_t* e, const int32_t* kind, const int32_t* param) {
    if (!e || !e->has_env || !kind) return set_error(RAMP_ERR_BAD_ARG, "no environment or no agent kinds");
    EnvDev& v = e->env;
    for (int b = 0; b < v.B; ++b)
        if (kind[b] < 0 || kind[b] >= RAMP_AGENT_COUNT) return set_error(RAMP_ERR_BAD_ARG, "episode %d: unknown agent kind %d", b, kind[b]);
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    CUDA_TRY(cudaMemcpy(v.agent_kind, kind, sizeof(int32_t) * v.B, cudaMemcpyHostToDevice));
    if (param) CUDA_TRY(cudaMemcpy(v.agent_param, param, sizeof(int32_t) * v.B, cudaMemcpyHostToDevice));
    else CUDA_TRY(cudaMemset(v.agent_param, 0, sizeof(int32_t) * v.B));
    e->env_agents_set = true;
    return RAMP_OK;
}

int ramp_env_agent_act(ramp_engine_t* e, uint64_t seed) {
    if (!e || !e->has_env) return set_error(RAMP_ERR_BAD_ARG, "no environment");
    if (!e->env_agents_set) return set_error(RAMP_ERR_BAD_ARG, "no agents: call ramp_env_set_agents first");
    const EnvDev& v = e->env;
    CUDA_TRY(cudaSetDevice(e->cfg.device));
    ramp_env_agent_kernel<<<(v.B + 127) / 128, 128, 0, e->stream.get()>>>(v, e->ep, (unsigned long long)seed);
    e->launches++;
    CUDA_TRY(cudaGetLastError());
    return RAMP_OK;
}

}  // extern "C"
