// ramp_lookahead_thread.cuh -- _run_lookahead (RCE:379-467) on QUOTIENT templates: ONE THREAD per lookahead.
//
// ramp_register_template folds every lowered job by its symmetries (ramp_quotient.cpp): the bench's ResNet-50-like job
// is 330 op classes and 887-1,413 dep entries at every partition degree, and its ready frontiers hold 0-6 items per
// tick.  There is nothing left for a warp to share, so each lookahead runs on ONE lane, scalar, with no shuffles,
// ballots, atomics or barriers in the tick loop:
//
//   * a CTA is a sim warp and a ledger warp (below); it pulls CHUNKS of up to 32 work items that use the same template
//     (ramp_bucket_kernel groups the step's memo misses by template), so the sim lanes run the same instruction stream over
//     the same template -- no divergence, and every template read is a shared-memory broadcast;
//   * the template blob (header + op records + rows + thresholds + out-entry records) is copied into shared
//     memory ONCE per chunk with a bulk async copy (cp.async.bulk -> UBLKCP, completion on an mbarrier), so a tick never
//     waits for L2;
//   * per-lane state is lane-interleaved in shared memory ([slot][lane]: conflict-free): u16 parent counters per op
//     class, the ready-op / ready-flow / ready-non-flow frontiers (first OCAP / FCAP / NFCAP entries; the rest spills to an
//     HBM slab laid out the same way), and small per-worker-group / per-channel-group winner tables.
//
// Per tick (letters as in SURVEY.md 3.3; same arithmetic, same order as ramp_lookahead_kernel):
//   A,B  winners among the ready op classes per worker group (largest rank key), t_op = min remaining, active workers =
//        sum of the winners' class sizes                                                        (RCE:562-606, 44-67, 709-715)
//   C    a ready non-flow dep makes this a zero-length tick that completes exactly the non-flows  (RCE:412-422, 520-540, 718-731)
//   D    else t_comm = min remaining over the per-channel-group winners among the ready flows     (RCE:608-663)
//   E    tick = min(t_op, t_comm)                                                                (RCE:426)
//   H    every ready flow: rem -= min(tick, rem); == 0 -> its child class's counter += entry size; the class is readied
//        when the counter passes through its threshold (n_parents x class size)                 (RCE:733-775, JOB:525-536)
//   G    winning op classes tick; == 0 -> completed, their out-entries become ready (first ticked next tick, RCE:429)
//   I,J  t / comm / comp, the utilisation term and the trace, f64, tick order                    (RCE:442-445, 777-791, 830-832)
//
// Only E..H and the frontier updates feed the next tick; I and J are accounting.  They run on a second warp: a CTA is two
// warps, and lane k of warp 0 (the SIM lane) and lane k of warp 1 (the LEDGER lane) share work item chunk * 32 + k.  The sim
// lane appends one record per tick {tick, n_active, flows ticked} to its ring in shared memory and publishes its record count
// every RAMP_T_PUB ticks; the ledger lane replays the records with the same f64 operations in the same order (bit-identical
// results), writes the trace, and runs the epilogue.  The sim warp's tick loop keeps no FP64 but the survivors' subtraction.
#pragma once

namespace ramp {

#ifndef RAMP_T_OCAP
#define RAMP_T_OCAP 8       // ready op classes kept in shared memory per lane
#endif
#ifndef RAMP_T_FCAP
#define RAMP_T_FCAP 16      // ready flow entries kept in shared memory per lane
#endif
#ifndef RAMP_T_FASTF
#define RAMP_T_FASTF 6      // frontiers of up to this many flow entries (and 2 op classes) run the register-resident path
#endif
#ifndef RAMP_T_NFCAP
#define RAMP_T_NFCAP 8      // ready non-flow entries kept in shared memory per lane
#endif
#define RAMP_T_WCAP 8       // worker groups with a per-lane winner table (more: pairwise comparison)
#define RAMP_T_CCAP 32      // channel groups with a per-lane winner table: the most a resident template may have
#ifndef RAMP_T_RING
#define RAMP_T_RING 32      // tick records per lane in the sim -> ledger ring (a power of two)
#endif
#ifndef RAMP_T_PUB
#define RAMP_T_PUB 8        // the sim lane publishes its record count every this many ticks (a power of two, <= RAMP_T_RING)
#endif
// the small-frontier path reads the first RAMP_T_FASTF flow entries and 2 op classes straight from shared memory, and every
// list keeps at least one entry there
static_assert(RAMP_T_FCAP >= RAMP_T_FASTF && RAMP_T_OCAP >= 2 && RAMP_T_NFCAP >= 1, "shared-memory capacities below the small-frontier path");
// RAMP_T_LEDGER_NS (off in the normal build): the ledger lane sleeps that many nanoseconds per record it consumes, so it stays
// behind its sim lane and the sim lane's ring-full wait runs on every template with enough ticks (tests/test_gpu_thread_kernel.py)
#define RAMP_T_DONE 0x80000000u   // set in the published count with the sim lane's last record
#define RAMP_THREAD_CTA 64  // threads of a thread-kernel CTA: the sim warp and the ledger warp

// header of a resident template blob (the blob is what the bulk copy moves: 16-byte aligned, size a multiple of 16)
struct ResHeader {
    int32_t n_ops, n_deps, n_workers, n_channels;      // classes, entries, worker groups, channel groups
    int32_t n_src, num_training_steps, orig_workers, _pad0;
    uint32_t kmask, cmask, imask, _pad1;               // dep word lo: key | SET of channel groups << cshift (empty: no channel);
    int32_t cshift, fshift, ishift, dshift;            // dep word hi: flow | inc << 1 | child << dshift  (fshift = 0, ishift = 1)
    int32_t off_op_row, off_op_thr, off_out, off_src;  // byte offsets from the blob start (op records follow the header)
    int32_t total_bytes, _pad2, _pad3, _pad4;
};
static_assert(sizeof(ResHeader) == 96, "resident header is 96 bytes");

struct ChunkDesc { int32_t template_id, count; };      // up to 32 work items of one template; items at [chunk * 32 + lane]
static_assert((RAMP_T_RING & (RAMP_T_RING - 1)) == 0 && (RAMP_T_PUB & (RAMP_T_PUB - 1)) == 0 && RAMP_T_PUB <= RAMP_T_RING,
              "ring and publish interval are powers of two");

// recorded by the first lookahead of a template that completes (deterministic per template): lets later ones write their trace
// in place and keep every list in shared memory
struct __align__(16) TemplateHints { int32_t n_ticks, max_o, max_f, max_nf; };   // read / written as ONE 16-byte access


struct ThreadArgs {
    const TemplateDev* templates;
    const ChunkDesc* chunks;
    const int32_t* n_chunks;        // device-side count
    int32_t* cursor;                // device-side chunk cursor (persistent CTAs pull chunks)
    const WorkItem* items;          // [chunk][32]
    unsigned char* scratch;         // [gridDim.x][scratch_stride]: per-CTA spill + temp trace
    uint64_t scratch_stride;
    ResultSlots res;
    TracePool pool;
    int32_t trace_cap;
    int32_t tmpl_cap;               // bytes of shared memory reserved for the template blob
    int32_t n_cap;                  // parent-counter slots per lane in shared memory
    int32_t spill_ops, spill_deps;  // per-lane spill capacities (entries) in the HBM slab
    MemoStats* stats;
    TemplateHints* hints;           // [max_templates], zero = nothing recorded yet
    double* hint_jct;               // [max_templates] job completion time the first lookahead of the template found (0 = none):
                                    //   lets later ones accumulate the utilisation inside the tick loop (RCE:830-832 divides by it)
};

__host__ __device__ inline size_t thread_smem_bytes(int tmpl_cap, int n_cap) {
    size_t per_lane = (size_t)RAMP_T_RING * 16 + (size_t)RAMP_T_FCAP * 16 + (size_t)RAMP_T_OCAP * 20 + (size_t)RAMP_T_NFCAP * 4
                      + (size_t)(RAMP_T_WCAP + RAMP_T_CCAP) * 4 + (size_t)n_cap * 2;
    return (size_t)tmpl_cap + 32 * per_lane + 64;
}
__host__ __device__ inline uint64_t thread_scratch_bytes(int spill_ops, int spill_deps, int trace_cap) {
    // per lane: ops spill (record 16 + index 4), flows spill (16), non-flow spill (4), temp trace (tick 8 + n 4)
    const uint64_t per_lane = (uint64_t)spill_ops * 20 + (uint64_t)spill_deps * 20 + (uint64_t)trace_cap * 12;
    return align_up(per_lane * 32, 256);
}

// ---------------------------------------------------------------------------------------------------
// groups a step's resident work items by template: chunks of up to 32 items of one template (single CTA)
struct BucketArgs {
    const WorkItem* items;          // unsorted memo misses whose template is resident
    int32_t* n_items;               // zeroed on exit (the next step's plan kernel appends from 0)
    int32_t n_templates;
    int32_t* tcount;                // [n_templates + 1] zero on entry, zero on exit
    int32_t* tbase;                 // [n_templates + 1] scratch: first chunk of each template
    WorkItem* chunk_items;          // [max_chunks][32]
    ChunkDesc* chunks;              // [max_chunks]
    int32_t* n_chunks;
    int32_t* cursor;                // reset to 0 here
    int32_t* rank;                  // [B] scratch
};

__global__ void __launch_bounds__(1024) ramp_bucket_kernel(const BucketArgs a) {
    __shared__ int s_scan[1024];
    __shared__ int s_carry;
    const int n = *a.n_items;
    const int tid = threadIdx.x;
    for (int i = tid; i < n; i += blockDim.x) a.rank[i] = atomicAdd(&a.tcount[a.items[i].template_id], 1);
    if (tid == 0) s_carry = 0;
    __syncthreads();
    // exclusive scan of chunks-per-template, 1024 templates per round
    for (int base = 0; base < a.n_templates; base += blockDim.x) {
        const int t = base + tid;
        const int cnt = (t < a.n_templates) ? a.tcount[t] : 0;
        const int nch = (cnt + 31) >> 5;
        s_scan[tid] = nch;
        __syncthreads();
        for (int o = 1; o < (int)blockDim.x; o <<= 1) {
            const int v = (tid >= o) ? s_scan[tid - o] : 0;
            __syncthreads();
            s_scan[tid] += v;
            __syncthreads();
        }
        const int excl = s_carry + s_scan[tid] - nch;
        if (t < a.n_templates) {
            a.tbase[t] = excl;
            for (int k = 0; k < nch; ++k) {
                ChunkDesc d; d.template_id = t; d.count = (cnt - 32 * k < 32) ? (cnt - 32 * k) : 32;
                a.chunks[excl + k] = d;
            }
        }
        __syncthreads();
        if (tid == blockDim.x - 1) s_carry += s_scan[tid];
        __syncthreads();
    }
    for (int i = tid; i < n; i += blockDim.x) {
        const WorkItem it = a.items[i];
        const int r = a.rank[i];
        a.chunk_items[(size_t)(a.tbase[it.template_id] + (r >> 5)) * 32 + (r & 31)] = it;
    }
    __syncthreads();
    for (int t = tid; t < a.n_templates; t += blockDim.x) a.tcount[t] = 0;
    if (tid == 0) { *a.n_chunks = s_carry; *a.cursor = 0; *a.n_items = 0; }
}

// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Lane-interleaved per-lane lists (element k of this lane at base[k * 32 + lane]).  SPILL: entries past the shared-memory
// capacity live in the CTA's HBM slab; !SPILL: the template's recorded frontier sizes (TemplateHints) fit the capacity.
//   ready op class   {remaining.lo, remaining.hi, key, worker group | class size << 16} + its class index
//   ready flow entry {remaining.lo, remaining.hi, dep word lo (key | set of channel groups << cshift), dep word hi (flow | inc << 1 | child << dshift)}
//   ready non-flow   dep word hi
// nothing the tick loop needs about a ready item is behind a second load
template <bool SPILL>
struct LaneOps {
    int4* a_sm; int32_t* i_sm; int4* a_gl; int32_t* i_gl; int lane;
    __device__ __forceinline__ int4 rec(int k) const {
        if (!SPILL || k < RAMP_T_OCAP) return a_sm[k * 32 + lane];
        return a_gl[(size_t)(k - RAMP_T_OCAP) * 32 + lane];
    }
    __device__ __forceinline__ int idx(int k) const {
        if (!SPILL || k < RAMP_T_OCAP) return i_sm[k * 32 + lane];
        return i_gl[(size_t)(k - RAMP_T_OCAP) * 32 + lane];
    }
    __device__ __forceinline__ void put(int k, const int4 r, int i) const {
        if (!SPILL || k < RAMP_T_OCAP) { a_sm[k * 32 + lane] = r; i_sm[k * 32 + lane] = i; }
        else { a_gl[(size_t)(k - RAMP_T_OCAP) * 32 + lane] = r; i_gl[(size_t)(k - RAMP_T_OCAP) * 32 + lane] = i; }
    }
};
template <bool SPILL>
struct LaneFlows {
    int4* sm; int4* gl; int lane;
    __device__ __forceinline__ int4 get(int k) const {
        if (!SPILL || k < RAMP_T_FCAP) return sm[k * 32 + lane];
        return gl[(size_t)(k - RAMP_T_FCAP) * 32 + lane];
    }
    __device__ __forceinline__ void put(int k, const int4 v) const {
        if (!SPILL || k < RAMP_T_FCAP) sm[k * 32 + lane] = v; else gl[(size_t)(k - RAMP_T_FCAP) * 32 + lane] = v;
    }
};
template <bool SPILL>
struct LaneNF {
    uint32_t* sm; uint32_t* gl; int lane;
    __device__ __forceinline__ uint32_t get(int k) const {
        if (!SPILL || k < RAMP_T_NFCAP) return sm[k * 32 + lane];
        return gl[(size_t)(k - RAMP_T_NFCAP) * 32 + lane];
    }
    __device__ __forceinline__ void put(int k, uint32_t v) const {
        if (!SPILL || k < RAMP_T_NFCAP) sm[k * 32 + lane] = v; else gl[(size_t)(k - RAMP_T_NFCAP) * 32 + lane] = v;
    }
};

// Remaining times are non-negative doubles (validated and canonicalised to +0 at registration): their u64 bit patterns order like
// the values, so every comparison of the tick loop -- winners' minimum, tick = min(t_comm, t_op), "did it complete" -- is a 64-bit
// INTEGER comparison (two ISETP) instead of an FP64 one: DSETP / DADD results come back through the long scoreboard, so FP64
// compares on the control path stall the tick loop; only the subtraction of the survivors and the three accumulators stay FP64,
// off the control path.
//   x -= min(tick, x) == 0  (JOB:555-556, 561-562)  <=>  x <= tick   (x > tick >= 0 gives x - tick > 0: no underflow to zero)
typedef unsigned long long u64_t;
__device__ __forceinline__ u64_t rem_bits(const int4& r) { return ((u64_t)(uint32_t)r.y << 32) | (u64_t)(uint32_t)r.x; }

// ---------------------------------------------------------------------------------------------------
// sim -> ledger ring: per lane, RAMP_T_RING records {tick.lo, tick.hi, n_active, flows ticked} at ring[slot * 32 + lane]; the
// sim lane publishes how many it has written (release), the ledger lane how many it has consumed (acquire / release pairs)
__device__ __forceinline__ void st_release_cta(uint32_t* p, uint32_t v) {
    asm volatile("st.release.cta.shared::cta.u32 [%0], %1;" ::"r"(smem_u32(p)), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_cta(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.cta.shared::cta.u32 %0, [%1];" : "=r"(v) : "r"(smem_u32(p)) : "memory");
    return v;
}

#ifdef RAMP_TICK_CLOCKS
// Cycle ledger of the sim lane, for measurement builds only (scripts/tick_cycles.py builds them; the library built without
// the switch has no trace of it).  Every sim lane reads clock() at the phase boundaries of each tick -- all lanes, so the
// warp stays converged -- and lane 0 adds the deltas to its CTA's row of ramp_tick_clocks, keyed by the tick's frontier
// shape.  A tick runs from its first stamp to the next tick's first stamp (or the loop's exit), so the phases add up to
// the tick loop's time.  The atomics are fire-and-forget reductions issued at the start of the next tick.
#define RAMP_TC_SHAPES 64       // ready op classes {0, 1, 2, >2} x ready flow entries {0..6, >6} x non-flow tick or not
#define RAMP_TC_PHASES 5        // A/B | D, E and the ring record | H | G | compaction, exit test and the loop's back edge
#define RAMP_TC_MAX_CTAS 1024
__device__ unsigned long long ramp_tick_clocks[RAMP_TC_MAX_CTAS][RAMP_TC_SHAPES][RAMP_TC_PHASES + 1];   // deltas, then ticks

struct TickClocks {
    uint32_t c[RAMP_TC_PHASES];
    int shape = -1;
    int lane;
    __device__ __forceinline__ void flush(uint32_t now) {
        if (shape >= 0 && lane == 0 && blockIdx.x < RAMP_TC_MAX_CTAS) {
            unsigned long long* t = ramp_tick_clocks[blockIdx.x][shape];
#pragma unroll
            for (int i = 0; i < RAMP_TC_PHASES; ++i) atomicAdd(t + i, (unsigned long long)(((i + 1 < RAMP_TC_PHASES) ? c[i + 1] : now) - c[i]));
            atomicAdd(t + RAMP_TC_PHASES, 1ull);
        }
    }
    __device__ __forceinline__ void begin(int nO, int nF, bool nf) {
        const uint32_t now = (uint32_t)clock();
        flush(now);
        shape = ((nO > 2 ? 3 : nO) * 8 + (nF > 6 ? 7 : nF)) * 2 + (nf ? 1 : 0);
        c[0] = now;
    }
    __device__ __forceinline__ void stamp(int i) { c[i] = (uint32_t)clock(); }
    __device__ __forceinline__ void finish() { flush((uint32_t)clock()); }
};
#define RAMP_TC(...) __VA_ARGS__
#else
#define RAMP_TC(...)
#endif

struct SimFinal { int status, tick_no, max_o, max_f, max_nf; };   // what the sim lane hands over with its last record

struct LedgerFeed {                   // the sim lane's end of its ring
    int4* ring; uint32_t* head; const uint32_t* tail; SimFinal* fin; int lane;
    uint32_t n, room;                 // records written; the first record number that has no free slot yet
    __device__ __forceinline__ void put(const u64_t tick_b, const int n_active, const bool flows) {
        if (n == room) {              // ring full: publish everything, then wait for the ledger lane to free a slot
            st_release_cta(head, n);
            uint32_t t;
            do { t = ld_acquire_cta(tail); } while (n - t >= RAMP_T_RING);
            room = t + RAMP_T_RING;
        }
        ring[(n & (RAMP_T_RING - 1)) * 32 + lane] = make_int4((int)(uint32_t)tick_b, (int)(uint32_t)(tick_b >> 32), n_active, flows ? 1 : 0);
        ++n;
        if ((n & (RAMP_T_PUB - 1)) == 0u) st_release_cta(head, n);
    }
    __device__ __forceinline__ void finish(const SimFinal& f) {
        *fin = f;
        st_release_cta(head, n | RAMP_T_DONE);
    }
};

struct LaneCtx {                      // what one sim lane's lookahead works on
    const unsigned char* tm;         // template blob in shared memory
    int4* f_sm; int4* o_sm; uint32_t* nf_sm; int32_t* oi_sm; uint32_t* wk_sm; uint32_t* ck_sm; uint16_t* cnt_sm;
    int4* f_gl; int4* o_gl; uint32_t* nf_gl; int32_t* oi_gl;
    int4* ring; uint32_t* head; const uint32_t* tail; SimFinal* fin;   // this lane's ledger feed
    int tr_cap;                      // ticks the trace can hold: one more is RAMP_ST_TRACE_OVERFLOW and ends the lookahead
    int lane, n_cap;
};

// _run_lookahead for one sim lane: the tick loop (A-H, K, L); every tick goes to the ledger lane as one ring record, and the
// final status, tick count and largest frontiers follow the last one.  SPILL = false: every frontier fits its shared-memory
// capacity (TemplateHints).  A tick with at most 2 ready op classes and RAMP_T_FASTF ready flow entries (every tick of the
// usual quotient of a partitioned job) runs the small-frontier half; any other tick runs the general half, whose winners come
// from per-group tables.  Both halves share the steps defined ahead of the loop and the end of the tick.
template <bool SPILL>
__device__ __forceinline__ void thread_lookahead(const LaneCtx& x) {
    const int lane = x.lane;
    const ResHeader& H = *reinterpret_cast<const ResHeader*>(x.tm);
    const int4* op_rec = reinterpret_cast<const int4*>(x.tm + sizeof(ResHeader));                  // {cost.lo, cost.hi, key, worker | weight << 16}
    const int2* op_row = reinterpret_cast<const int2*>(x.tm + H.off_op_row);                        // {first, n flows | n non-flows << 16}
    const uint32_t* op_thr = reinterpret_cast<const uint32_t*>(x.tm + H.off_op_thr);
    const int4* out_rec = reinterpret_cast<const int4*>(x.tm + H.off_out);                          // ready-flow entries, as appended
    const int32_t* src_ops = reinterpret_cast<const int32_t*>(x.tm + H.off_src);
    const int N = H.n_ops, E = H.n_deps, W = H.n_workers, C = H.n_channels;
    const uint32_t kmask = H.kmask, imask = H.imask;
    const int csh = H.cshift, dsh = H.dshift;
    const bool tab_w = (W <= RAMP_T_WCAP);
    const LaneOps<SPILL> ops{x.o_sm, x.oi_sm, x.o_gl, x.oi_gl, lane};
    const LaneFlows<SPILL> flows{x.f_sm, x.f_gl, lane};
    const LaneNF<SPILL> nfs{x.nf_sm, x.nf_gl, lane};
    uint16_t* cnt = x.cnt_sm + lane;
    uint32_t* wk = x.wk_sm + lane;
    uint32_t* ck = x.ck_sm + lane;
    const double INF = __longlong_as_double(RAMP_INF_BITS);

    for (int i = 0; i < N && i < x.n_cap; ++i) cnt[i * 32] = 0;
    int nO = H.n_src, nF = 0, nNF = 0;
    // JOB:496-506: a completed class's out-entries become ready.  The blob stores them as ready-made frontier entries, flows
    // first, in descending key order (ramp_engine.cu, build_resident_blob).  The ready-flow frontier is kept in descending key
    // order too (entries of equal key adjacent), which is what the small-frontier half's one-pass channel winners need: the
    // class's flows are merged into it from the back -- a straight copy when the frontier is empty, the usual case -- and
    // every survivor compaction keeps the order.  Nothing else depends on the order of a frontier.
    auto complete_op = [&](const int op) {
        const int2 row = op_row[op];
        const int e_nf = row.x + (row.y & 0xffff), e_end = e_nf + (row.y >> 16);
        if (nF == 0) {
            _Pragma("unroll 1")
            for (int e = row.x; e < e_nf; ++e) { flows.put(nF, out_rec[e]); ++nF; }
        } else {
            int i = nF - 1, k = nF + (e_nf - row.x) - 1;
            nF = k + 1;
            _Pragma("unroll 1")
            for (int e = e_nf - 1; e >= row.x; --e, --k) {
                const int4 r = out_rec[e];
                const uint32_t key = (uint32_t)r.z & kmask;
                _Pragma("unroll 1")
                for (int4 f; i >= 0 && ((uint32_t)(f = flows.get(i)).z & kmask) < key; --i, --k) flows.put(k, f);
                flows.put(k, r);
            }
        }
        _Pragma("unroll 1")
        for (int e = e_nf; e < e_end; ++e) { nfs.put(nNF, (uint32_t)out_rec[e].w); ++nNF; }
    };
    for (int k = 0; k < nO; ++k) { const int op = src_ops[k]; ops.put(k, op_rec[op], op); }       // RCE:1334
    SimFinal R;
    R.tick_no = 0; R.max_o = nO; R.max_f = 0; R.max_nf = 0;
    R.status = (N <= x.n_cap) ? RAMP_ST_OK : RAMP_ST_TABLE_FULL;                                    // cannot happen (eligibility)
    int to_complete = N + E;              // ops and deps still to complete (JOB:549-551)
    LedgerFeed feed{x.ring, x.head, x.tail, x.fin, lane, 0u, (uint32_t)RAMP_T_RING};
    RAMP_TC(TickClocks tc; tc.lane = lane;)
    // the tick's state: t_op = smallest remaining time of the op winners and n_active = their class sizes (A, B), the tick
    // (E), and tailO, the end of the op-class frontier: classes readied in the tick are appended behind it (H, G)
    u64_t t_op = RAMP_INF_BITS, tick_b = 0ull;
    double tick = 0.0;
    int n_active = 0, tailO = nO;
    auto complete_dep = [&](const uint32_t hi) {                                                    // JOB:525-536
        const int child = (int)(hi >> dsh);
        const uint32_t inc = (hi >> 1) & imask;
        const uint32_t old = cnt[child * 32];
        const uint32_t thr = op_thr[child];
        const uint32_t neu = old + inc;
        cnt[child * 32] = (uint16_t)neu;
        if (old < thr && thr <= neu) { ops.put(tailO, op_rec[child], child); ++tailO; }             // JOB:531 for every member
    };
    // ---- E: the tick; its record goes to the ledger lane (I, J) ----
    auto take_tick = [&](const u64_t t_comm, const bool ticked_flows) {
        tick_b = (t_comm < t_op) ? t_comm : t_op;
        tick = __longlong_as_double((long long)tick_b);
        feed.put(tick_b, n_active, ticked_flows);
        if (R.tick_no >= x.tr_cap) R.status = RAMP_ST_TRACE_OVERFLOW;
        ++R.tick_no;
        RAMP_TC(tc.stamp(2);)
    };

    if (R.status == RAMP_ST_OK) for (;;) {       // left through ONE combined exit test per tick
        RAMP_TC(tc.begin(nO, nF, nNF > 0);)
        t_op = RAMP_INF_BITS;
        n_active = 0;
        tailO = nO;
        const bool any_nf = nNF > 0;
        int p = 0;                               // op classes left after G
        if (nF <= RAMP_T_FASTF && nO <= 2) {
            // ======== small frontiers (the usual case on a quotient): every ready item is loaded ONCE into registers and each
            // phase runs code specialised for the exact number of ready ops (0-2) and flows (0-6): winners by pairwise
            // comparison (no tables, any number of worker / channel groups), no loop or predication overhead ========
            static_assert(RAMP_T_FASTF == 6, "the dispatch below has cases for up to 6 ready flow entries");
            int4 fr[RAMP_T_FASTF], orr[2];
            int oi[2];
            bool ow0 = false, ow1 = false;
            // ---- A, B ----
            if (nO >= 1) {
                orr[0] = x.o_sm[lane]; oi[0] = x.oi_sm[lane];
                ow0 = true;
                if (nO == 2) {
                    orr[1] = x.o_sm[32 + lane]; oi[1] = x.oi_sm[32 + lane];
                    ow1 = true;
                    if (((orr[0].w ^ orr[1].w) & 0xffff) == 0) { if ((uint32_t)orr[0].z > (uint32_t)orr[1].z) ow1 = false; else ow0 = false; }
                    if (ow1) { t_op = rem_bits(orr[1]); n_active = (int)((uint32_t)orr[1].w >> 16); }
                }
                if (ow0) { const u64_t r0 = rem_bits(orr[0]); t_op = (r0 < t_op) ? r0 : t_op; n_active += (int)((uint32_t)orr[0].w >> 16); }
            }
            RAMP_TC(tc.stamp(1);)
            // ---- C, D, E, I, J, H: dispatched ONCE on the number of ready flow entries; each case is straight-line code
            // without a branch but the completions: D and H are one pass each over the key-ordered frontier ----
            auto flow_tick = [&](auto nf_tag) {
                constexpr int NF = decltype(nf_tag)::value;
#pragma unroll
                for (int k = 0; k < NF; ++k) fr[k] = x.f_sm[k * 32 + lane];
                // D: the entry wins on a channel group of its set unless a ready entry with a larger key lies on that group
                // too (an empty set -- no channel -- never wins, it only ticks).  In key order the larger keys are the entries
                // before the entry's run of equal keys, so one pass with the groups they claim gives the pairwise rule.
                u64_t t_comm = RAMP_INF_BITS;
                uint32_t seen = 0u, claimed = 0u;       // groups of the entries so far / of those with a larger key
#pragma unroll
                for (int k = 0; k < NF; ++k) {
                    const uint32_t gm = (uint32_t)fr[k].z >> csh;
                    if (k > 0) claimed = (((uint32_t)fr[k].z & kmask) != ((uint32_t)fr[k - 1].z & kmask)) ? seen : claimed;
                    const u64_t rem = rem_bits(fr[k]);
                    t_comm = ((gm & ~claimed) != 0u && rem < t_comm) ? rem : t_comm;
                    seen |= gm;
                }
                take_tick(t_comm, true);
                // H: every entry ticks (JOB:561-562); survivors are compacted to the front in order, completed entries go to
                // the back of the old slots, both by ONE store whose slot is selected
                int pf = 0, nd = 0;             // survivors; completed entries: the first one's dep word hi in hd0, the
                uint32_t hd0 = 0u;              // others at slots NF - 2, NF - 3, ...
#pragma unroll
                for (int k = 0; k < NF; ++k) {
                    const u64_t rb = rem_bits(fr[k]);
                    const bool done = rb <= tick_b;
                    const double r2 = __dsub_rn(__longlong_as_double((long long)rb), tick);
                    int4 f = fr[k];
                    f.x = __double2loint(r2); f.y = __double2hiint(r2);
                    hd0 = (done && nd == 0) ? (uint32_t)f.w : hd0;
                    x.f_sm[(done ? NF - 1 - nd : pf) * 32 + lane] = f;
                    pf += done ? 0 : 1;
                    nd += done ? 1 : 0;
                }
                nF = pf;
                // the completed entries' children, in slot order
                if (nd != 0) {
                    complete_dep(hd0);
                    _Pragma("unroll 1")
                    for (int d = 1; d < nd; ++d) complete_dep((uint32_t)x.f_sm[(NF - 1 - d) * 32 + lane].w);
                    to_complete -= nd;
                }
            };
            // by frequency on the quotient of a partitioned job: one ready flow entry, a non-flow tick, none, two, ...
            if (any_nf) {                                           // zero-length tick that completes the ready non-flow deps
                take_tick(0ull, false);
                _Pragma("unroll 1")
                for (int k = 0; k < nNF; ++k) complete_dep(nfs.get(k));
                to_complete -= nNF;
                nNF = 0;
            } else {
                // a chain of compare-and-branch, most frequent count first; the empty asm keeps the compiler from folding the chain
                // back into a jump table (constant-bank load + indirect branch on the critical path of every tick)
                auto opaque = [](int v) { asm volatile("" : "+r"(v)); return v; };
                if (opaque(nF) == 1) flow_tick(std::integral_constant<int, 1>{});
                else if (opaque(nF) == 0) take_tick(RAMP_INF_BITS, false);
                else if (opaque(nF) == 2) flow_tick(std::integral_constant<int, 2>{});
                else if (opaque(nF) == 3) flow_tick(std::integral_constant<int, 3>{});
                else if (opaque(nF) == 4) flow_tick(std::integral_constant<int, 4>{});
                else if (opaque(nF) == 5) flow_tick(std::integral_constant<int, 5>{});
                else flow_tick(std::integral_constant<int, 6>{});
            }
            RAMP_TC(tc.stamp(3);)
            // ---- G ----
            auto tick_op = [&](int4 r, const int op, const bool win) {
                if (win) {                                                                          // this tick's winner
                    const u64_t rb = rem_bits(r);
                    if (rb <= tick_b) {                                                             // JOB:555-556
                        --to_complete;
                        complete_op(op);
                        return;
                    }
                    const double rem = __dsub_rn(__longlong_as_double((long long)rb), tick);
                    r.x = __double2loint(rem); r.y = __double2hiint(rem);
                }
                x.o_sm[p * 32 + lane] = r; x.oi_sm[p * 32 + lane] = op; ++p;
            };
            if (nO >= 1) {
                tick_op(orr[0], oi[0], ow0);
                if (nO == 2) tick_op(orr[1], oi[1], ow1);
            }
        } else {
            // ---- A, B: winners per worker group: largest key; t_op = min of their remaining times ----
            if (nO > 0) {
                if (tab_w) {
                    _Pragma("unroll 1")
                    for (int w = 0; w < W; ++w) wk[w * 32] = 0u;
                    _Pragma("unroll 1")
                    for (int k = 0; k < nO; ++k) {
                        const int4 r = ops.rec(k);
                        const int w = r.w & 0xffff;
                        if ((uint32_t)r.z > wk[w * 32]) wk[w * 32] = (uint32_t)r.z;
                    }
                    _Pragma("unroll 1")
                    for (int k = 0; k < nO; ++k) {
                        const int4 r = ops.rec(k);
                        if (wk[(r.w & 0xffff) * 32] == (uint32_t)r.z) {
                            const u64_t rem = rem_bits(r);
                            t_op = (rem < t_op) ? rem : t_op;
                            n_active += (int)((uint32_t)r.w >> 16);
                        }
                    }
                } else {
                    // more worker groups than table slots: pairwise comparison; the winners are marked in bit 31 of the key
                    // (keys are ranks <= N < 2^31) for phase G, which clears the mark
                    _Pragma("unroll 1")
                    for (int k = 0; k < nO; ++k) {
                        int4 r = ops.rec(k);
                        bool win = true;
                        _Pragma("unroll 1")
                        for (int j = 0; j < nO && win; ++j) {
                            const int4 r2 = ops.rec(j);
                            if ((r2.w & 0xffff) == (r.w & 0xffff) && ((uint32_t)r2.z & 0x7fffffffu) > (uint32_t)r.z) win = false;
                        }
                        if (win) {
                            const u64_t rem = rem_bits(r);
                            t_op = (rem < t_op) ? rem : t_op;
                            n_active += (int)((uint32_t)r.w >> 16);
                            r.z = (int)((uint32_t)r.z | 0x80000000u);
                            ops.put(k, r, ops.idx(k));
                        }
                    }
                }
            }
            RAMP_TC(tc.stamp(1);)
            // ---- C, D ----
            u64_t t_comm = 0ull;
            if (!any_nf) {
                t_comm = RAMP_INF_BITS;
                if (nF > 0) {
                    // per-group table: largest key among the ready entries whose set contains the group (a resident template
                    // has at most RAMP_T_CCAP channel groups: build_resident_blob)
                    _Pragma("unroll 1")
                    for (int q = 0; q < C; ++q) ck[q * 32] = 0u;
                    _Pragma("unroll 1")
                    for (int k = 0; k < nF; ++k) {
                        const uint32_t lo = (uint32_t)flows.get(k).z;
                        const uint32_t key = lo & kmask;
                        uint32_t m = lo >> csh;
                        while (m) { const int q = __ffs((int)m) - 1; m &= m - 1u; if (key > ck[q * 32]) ck[q * 32] = key; }
                    }
                    _Pragma("unroll 1")
                    for (int k = 0; k < nF; ++k) {
                        const int4 f = flows.get(k);
                        const uint32_t key = (uint32_t)f.z & kmask;
                        uint32_t m = (uint32_t)f.z >> csh;
                        bool win = false;
                        while (m && !win) { const int q = __ffs((int)m) - 1; m &= m - 1u; win = ck[q * 32] == key; }
                        if (win) { const u64_t rem = rem_bits(f); t_comm = (rem < t_comm) ? rem : t_comm; }
                    }
                }
            }
            take_tick(t_comm, (!any_nf) && (nF > 0));
            // ---- H ----
            if (any_nf) {
                _Pragma("unroll 1")
                for (int k = 0; k < nNF; ++k) complete_dep(nfs.get(k));
                to_complete -= nNF;
                nNF = 0;
            } else {
                int pf = 0;
                _Pragma("unroll 1")
                for (int k = 0; k < nF; ++k) {
                    int4 f = flows.get(k);
                    const u64_t rb = rem_bits(f);
                    if (rb <= tick_b) { complete_dep((uint32_t)f.w); --to_complete; }            // JOB:561-562
                    else {
                        const double r2 = __dsub_rn(__longlong_as_double((long long)rb), tick);
                        f.x = __double2loint(r2); f.y = __double2hiint(r2); flows.put(pf, f); ++pf;
                    }
                }
                nF = pf;
            }
            RAMP_TC(tc.stamp(3);)
            // ---- G ----
            _Pragma("unroll 1")
            for (int k = 0; k < nO; ++k) {
                int4 r = ops.rec(k);
                const int op = ops.idx(k);
                bool win;
                if (tab_w) win = wk[(r.w & 0xffff) * 32] == (uint32_t)r.z;
                else { win = r.z < 0; r.z &= 0x7fffffff; }
                if (win) {                                                                          // this tick's winner
                    const u64_t rb = rem_bits(r);
                    if (rb <= tick_b) {                                                             // JOB:555-556
                        --to_complete;
                        complete_op(op);
                        continue;
                    }
                    const double rem = __dsub_rn(__longlong_as_double((long long)rb), tick);
                    r.x = __double2loint(rem); r.y = __double2hiint(rem);
                }
                ops.put(p, r, op); ++p;
            }
        }
        RAMP_TC(tc.stamp(4);)
        // the classes readied in this tick go behind the p that are left
        if (tailO != nO) {
            _Pragma("unroll 1")
            for (int k = nO; k < tailO; ++k, ++p) { if (p != k) ops.put(p, ops.rec(k), ops.idx(k)); }
        }
        nO = p;
        if (SPILL) {                              // the sizes the fast path relies on next time (TemplateHints)
            R.max_o = (tailO > R.max_o) ? tailO : R.max_o;
            R.max_f = (nF > R.max_f) ? nF : R.max_f;
            R.max_nf = (nNF > R.max_nf) ? nNF : R.max_nf;
        }
        // ---- K, L ----
        if ((to_complete == 0) | ((uint32_t)(tick_b >> 32) == 0x7FF00000u) | (R.status != RAMP_ST_OK)) {
            if (to_complete != 0 && (uint32_t)(tick_b >> 32) == 0x7FF00000u) R.status = RAMP_ST_INFINITE_TICK;       // JOB:549-551 first, then RCE:462
            break;
        }
    }
    RAMP_TC(tc.finish();)
    feed.finish(R);
}

// ---------------------------------------------------------------------------------------------------
// The ledger lane: replays its sim lane's ticks in tick order -- t / comm / comp (RCE:434-445, 777-791), the utilisation term
// (RCE:830-832) and the trace element -- with the f64 operations the tick loop used to do itself, in the same order.
struct LedgerCtx {
    const int4* ring; const uint32_t* head; uint32_t* tail; int lane;
    int32_t* tr_n; double* tr_tick;  // trace destination: element k at [k * tr_stride]
    int tr_stride, tr_cap;
    double util_jct, util_dn;        // != 0: accumulate sum (n_active / util_dn) * (tick / util_jct) in tick order (RCE:830-832)
};
struct LedgerSums { double t, comm, comp, util; };

__device__ __forceinline__ LedgerSums ledger_run(const LedgerCtx& y) {
    LedgerSums S;
    S.t = 0.0; S.comm = 0.0; S.comp = 0.0; S.util = 0.0;
    const bool do_util = y.util_jct != 0.0;
    int util_last_n = -1;
    double util_last_q = 0.0;
    int tr_idx = 0;
    uint32_t k = 0;                       // records consumed
    for (;;) {
        const uint32_t h = ld_acquire_cta(y.head);
        const uint32_t end = h & ~RAMP_T_DONE;
        if (k == end) {
            if (h & RAMP_T_DONE) break;
            __nanosleep(64);              // the sim lane publishes every RAMP_T_PUB ticks (several microseconds): poll gently
            continue;
        }
        _Pragma("unroll 1")
        for (; k != end; ++k) {
            const int4 r = y.ring[(k & (RAMP_T_RING - 1)) * 32 + y.lane];
            const u64_t tick_b = rem_bits(r);
            const double tick = __longlong_as_double((long long)tick_b);
            const int n_active = r.z;
            if (r.w) S.comm = __dadd_rn(S.comm, tick);
            if (n_active > 0) {
                S.comp = __dadd_rn(S.comp, tick);
                // a tick with no active worker or no length adds +0.0 and is skipped (see the epilogue)
                if (do_util && tick_b != 0ull) {
                    if (n_active != util_last_n) { util_last_n = n_active; util_last_q = __ddiv_rn((double)n_active, y.util_dn); }
                    S.util = __dadd_rn(S.util, __dmul_rn(util_last_q, __ddiv_rn(tick, y.util_jct)));
                }
            }
            S.t = __dadd_rn(S.t, tick);
            if ((int)k < y.tr_cap) { y.tr_n[tr_idx] = n_active; y.tr_tick[tr_idx] = tick; tr_idx += y.tr_stride; }
#ifdef RAMP_T_LEDGER_NS
            __nanosleep(RAMP_T_LEDGER_NS);
#endif
        }
        st_release_cta(y.tail, k);
    }
    return S;
}

__global__ void __launch_bounds__(RAMP_THREAD_CTA) ramp_lookahead_thread_kernel(const ThreadArgs a) {
    extern __shared__ __align__(128) unsigned char smem_thr[];
    __shared__ __align__(8) unsigned long long mbar;
    __shared__ uint32_t s_head[32], s_tail[32];     // per lane: ring records the sim lane published / the ledger lane consumed
    __shared__ SimFinal s_fin[32];                   // per lane: the sim lane's status, tick count and largest frontiers
    __shared__ int32_t s_tr_cap[32];                 // per lane: ticks its trace holds (the ledger lane places the trace)
    __shared__ int4 s_chunk;                         // {chunk, template (-1: none left), count, -}
    __shared__ int4 s_hint;                          // TemplateHints of the chunk's template
    __shared__ double s_hint_jct;
    const int lane = threadIdx.x & 31;
    const bool is_sim = threadIdx.x < 32;           // warp 0: tick loops; warp 1: ledger lanes
    unsigned char* st = smem_thr + a.tmpl_cap;                      // per-lane state, by decreasing alignment
    int4* ring = reinterpret_cast<int4*>(st);                                            // [RING][32]
    LaneCtx x;
    x.tm = smem_thr;                                                // template blob
    x.f_sm = ring + RAMP_T_RING * 32;                                                    // [FCAP][32]
    x.o_sm = x.f_sm + RAMP_T_FCAP * 32;                                                  // [OCAP][32]
    x.nf_sm = reinterpret_cast<uint32_t*>(x.o_sm + RAMP_T_OCAP * 32);                    // [NFCAP][32]
    x.oi_sm = reinterpret_cast<int32_t*>(x.nf_sm + RAMP_T_NFCAP * 32);                   // [OCAP][32]
    x.wk_sm = reinterpret_cast<uint32_t*>(x.oi_sm + RAMP_T_OCAP * 32);                   // [WCAP][32]
    x.ck_sm = x.wk_sm + RAMP_T_WCAP * 32;                                                // [CCAP][32]
    x.cnt_sm = reinterpret_cast<uint16_t*>(x.ck_sm + RAMP_T_CCAP * 32);                  // [n_cap][32]
    unsigned char* slab = a.scratch + (uint64_t)blockIdx.x * a.scratch_stride;
    x.f_gl = reinterpret_cast<int4*>(slab);                                              // [spill_deps][32]
    x.o_gl = x.f_gl + (size_t)a.spill_deps * 32;                                         // [spill_ops][32]
    double* tmp_tick = reinterpret_cast<double*>(x.o_gl + (size_t)a.spill_ops * 32);     // [trace_cap][32]
    x.nf_gl = reinterpret_cast<uint32_t*>(tmp_tick + (size_t)a.trace_cap * 32);          // [spill_deps][32]
    x.oi_gl = reinterpret_cast<int32_t*>(x.nf_gl + (size_t)a.spill_deps * 32);           // [spill_ops][32]
    int32_t* tmp_n = x.oi_gl + (size_t)a.spill_ops * 32;                                 // [trace_cap][32]
    x.ring = ring; x.head = &s_head[lane]; x.tail = &s_tail[lane]; x.fin = &s_fin[lane];
    x.lane = lane; x.n_cap = a.n_cap;

    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&mbar)));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    uint32_t phase = 0;
    int loaded = -1;

    for (;;) {
        // both warps are done with the previous chunk (the barrier below): order their generic-proxy accesses to the blob
        // before the async-proxy writes of a bulk copy into it
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        if (threadIdx.x == 0) {
            // the chunk, and what an earlier lookahead of its template recorded (number of ticks, largest frontiers,
            // completion time: deterministic per template), read ONCE so that both warps take the same path
            int4 cd = make_int4(0, -1, 0, 0), hv = make_int4(0, 0, 0, 0);
            double hj = 0.0;
            const int c = atomicAdd(a.cursor, 1);
            if (c < *a.n_chunks) {
                const ChunkDesc ch = a.chunks[c];
                cd = make_int4(c, ch.template_id, ch.count, 0);
                // n_ticks is the record's flag: acquired first, the rest of the record is read only when it is set
                const TemplateHints* hp = &a.hints[ch.template_id];
                int n_ticks = 0;
                asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(n_ticks) : "l"(&hp->n_ticks) : "memory");
                if (n_ticks > 0) {
                    hv = make_int4(n_ticks, __ldcg(&hp->max_o), __ldcg(&hp->max_f), __ldcg(&hp->max_nf));
                    hj = __ldcg(&a.hint_jct[ch.template_id]);
                }
            }
            s_chunk = cd; s_hint = hv; s_hint_jct = hj;
        }
        __syncthreads();
        const int4 cd = s_chunk;
        if (cd.y < 0) break;
        const int c = cd.x, tmpl = cd.y, count = cd.z;
        TemplateHints hint;
        { const int4 hv = s_hint; hint.n_ticks = hv.x; hint.max_o = hv.y; hint.max_f = hv.z; hint.max_nf = hv.w; }
        const double hj = s_hint_jct;
        const TemplateDev& TD = a.templates[tmpl];
        if (tmpl != loaded) {
            if (threadIdx.x == 0) {
                const uint32_t bytes = (uint32_t)TD.res_bytes;
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(&mbar)), "r"(bytes) : "memory");
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             ::"r"(smem_u32(smem_thr)), "l"(TD.res_blob), "r"(bytes), "r"(smem_u32(&mbar)) : "memory");
            }
            asm volatile(
                "{\n"
                ".reg .pred p;\n"
                "RAMP_WAIT_%=:\n"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
                "@p bra RAMP_DONE_%=;\n"
                "bra RAMP_WAIT_%=;\n"
                "RAMP_DONE_%=:\n"
                "}\n" ::"r"(smem_u32(&mbar)), "r"(phase) : "memory");
            phase ^= 1u;
            loaded = tmpl;
        }
        // with the hints the trace goes straight to an exactly-sized pool allocation and no list can leave shared memory
        const bool fast = hint.n_ticks > 0 && hint.n_ticks <= a.trace_cap && hint.max_o <= RAMP_T_OCAP && hint.max_f <= RAMP_T_FCAP
                          && hint.max_nf <= RAMP_T_NFCAP;
        const ResHeader& H = *reinterpret_cast<const ResHeader*>(x.tm);
        const bool active = lane < count;

        // ---- ledger lane, before the tick loop: trace destination and utilisation inputs ----
        LedgerCtx y;
        WorkItem item;
        long long off = -1;
        int status0 = RAMP_ST_OK, nmw = 0, num_training_steps = 0, n_ops = 0, n_deps = 0;
        const bool direct = fast && a.pool.top != nullptr;              // trace written in place
        if (!is_sim) {
            s_head[lane] = 0u; s_tail[lane] = 0u;
            if (active) {
                item = a.items[(size_t)c * 32 + lane];
                num_training_steps = H.num_training_steps; n_ops = H.n_ops; n_deps = H.n_deps;   // header fields the epilogue needs
                if (direct) {
                    const unsigned long long o = atomicAdd(a.pool.top, (unsigned long long)hint.n_ticks);
                    if (o + (unsigned long long)hint.n_ticks <= a.pool.len) off = (long long)o; else status0 = RAMP_ST_TRACE_OVERFLOW;
                }
                y.ring = ring; y.head = &s_head[lane]; y.tail = &s_tail[lane]; y.lane = lane;
                if (off >= 0) { y.tr_n = a.pool.n_active + off; y.tr_tick = a.pool.tick + off; y.tr_stride = 1; y.tr_cap = hint.n_ticks; }
                else { y.tr_n = tmp_n + lane; y.tr_tick = tmp_tick + lane; y.tr_stride = 32; y.tr_cap = a.trace_cap; }
                s_tr_cap[lane] = y.tr_cap;
                // utilisation inside the tick loop when an earlier lookahead of the template left its completion time
                nmw = item.n_mounted_workers > 0 ? item.n_mounted_workers : H.orig_workers;
                y.util_jct = (fast && hj > 0.0 && !isinf(hj)) ? hj : 0.0;
                {   // keep the conversion out of the loop (the compiler re-materialised it there: one I2F.F64 per tick)
                    double dn = (double)nmw;
                    asm volatile("" : "+d"(dn));
                    y.util_dn = dn;
                }
            }
        }
        __syncthreads();              // ring counters reset and s_tr_cap set; every thread has read s_chunk / s_hint

        if (is_sim) {
            if (active) {
                x.tr_cap = s_tr_cap[lane];
                // one instantiation per line: scripts/tick_cycles.py finds each one's SASS by the line it is inlined at
                if (fast) thread_lookahead<false>(x);
                else thread_lookahead<true>(x);
            }
            continue;
        }
        if (!active) continue;
        const LedgerSums S = ledger_run(y);
        const SimFinal R = s_fin[lane];           // written before the DONE count ledger_run acquired
        int status = (R.status == RAMP_ST_OK) ? status0 : R.status;
        if (direct && status == RAMP_ST_OK && R.tick_no != hint.n_ticks) status = RAMP_ST_TRACE_OVERFLOW;   // cannot happen
        if (!fast && status == RAMP_ST_OK) {
            // every lookahead of the template writes the same values, from this CTA or from one of another lookahead window
            // running at the same time; n_ticks (> 0) is stored last with release semantics, so a reader that acquires it sees
            // the whole record
            TemplateHints* hp = &a.hints[tmpl];
            hp->max_o = R.max_o; hp->max_f = R.max_f; hp->max_nf = R.max_nf;
            a.hint_jct[tmpl] = __dmul_rn(S.t, (double)num_training_steps);
            asm volatile("st.release.gpu.global.b32 [%0], %1;" :: "l"(&hp->n_ticks), "r"(R.tick_no) : "memory");
        }

        // ---- results (RCE:450-452) ----
        const int n_rec = R.tick_no < y.tr_cap ? R.tick_no : y.tr_cap;
        const double steps = (double)num_training_steps;
        const double jct = __dmul_rn(S.t, steps);
        const bool can_util = (status == RAMP_ST_OK);
        // the in-loop sum divided by the recorded completion time: valid when this lookahead found the very same one
        const bool util_done = can_util && y.util_jct != 0.0 && jct == y.util_jct;
        if (!direct && a.pool.top != nullptr) {
            const unsigned long long o = atomicAdd(a.pool.top, (unsigned long long)n_rec);
            if (o + (unsigned long long)n_rec <= a.pool.len) off = (long long)o;
            else if (status == RAMP_ST_OK) status = RAMP_ST_TRACE_OVERFLOW;
        }
        double util = util_done ? S.util : 0.0;
        if (!(util_done && (direct || off < 0))) {
            if (util_done) util = 0.0;                 // the loop below recomputes it while it copies the trace
            // RCE:830-832: util = sum over ticks, in tick order, of (n_active / n_mounted_workers) * (tick / jct).  A term
            // with n_active == 0 or tick == 0 is +0.0 (jct > 0 finite) and adding +0.0 leaves the non-negative sum as it
            // is, so those ticks are skipped (about two thirds of them); n_active / n_mounted_workers is re-used while
            // n_active repeats.  Same f64 operations on the same values for every term that can change the sum.
            const double dn = (double)nmw;
            const bool copy = (!direct) && off >= 0;
            int32_t* pn = copy ? a.pool.n_active + off : nullptr;
            double* pt = copy ? a.pool.tick + off : nullptr;
            const int32_t* sn = y.tr_n; const double* stt = y.tr_tick; const int sstr = y.tr_stride;
            const bool skip_zero = can_util && (jct > 0.0) && !isinf(jct);
            int last_n = -1;
            double last_q = 0.0;
#pragma unroll 4
            for (int k = 0; k < n_rec; ++k) {
                const int nk = sn[(size_t)k * sstr];
                const double tk = stt[(size_t)k * sstr];
                if (copy) { pn[k] = nk; pt[k] = tk; }
                if (!can_util) continue;
                if (skip_zero && (nk == 0 || tk == 0.0)) continue;
                if (nk != last_n) { last_n = nk; last_q = __ddiv_rn((double)nk, dn); }
                util = __dadd_rn(util, __dmul_rn(last_q, __ddiv_rn(tk, jct)));
            }
        }
        a.res.jct[item.slot] = jct;
        a.res.comm[item.slot] = __dmul_rn(S.comm, steps);
        a.res.comp[item.slot] = __dmul_rn(S.comp, steps);
        a.res.n_ticks[item.slot] = R.tick_no;
        a.res.util[item.slot] = can_util ? util : 0.0;
        a.res.util_nmw[item.slot] = can_util ? nmw : -1;
        a.res.trace_off[item.slot] = off;
        a.res.status[item.slot] = status;
        if (a.stats) {
            atomicAdd(&a.stats->lookaheads, 1ull);
            atomicAdd(&a.stats->alg_bytes, (unsigned long long)(TD.algorithmic_bytes_static + 12ull * (unsigned long long)R.tick_no));
            atomicAdd(&a.stats->quotient_bytes, (unsigned long long)(20ull * n_ops + 19ull * n_deps + 24ull + 12ull * (unsigned long long)R.tick_no));
        }
    }
}

}  // namespace ramp
