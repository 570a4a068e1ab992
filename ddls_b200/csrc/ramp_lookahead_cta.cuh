// ramp_lookahead_cta.cuh -- _run_lookahead (RCE:379-467) with ONE CTA (NW warps) per lookahead.
//
// Runs every lookahead whose template is not resident (its quotient blob does not fit shared memory, or
// RAMP_LOOKAHEAD_MODE=cta); the per-tick passes are spread over the CTA's warps so a single lookahead finishes sooner.
// The engine picks 256, 128 or 64 threads per CTA by how many such lookaheads a launch has (launch_lookaheads).
//
// The dep frontier is one list updated IN PLACE (completed entries are marked dead, ticks that freeze the flows write
// nothing) and compacted into the other buffer only when more than half of it is dead; newly ready deps are appended
// at its tail (first ticked next tick: the RCE:429 snapshot).  Per-tick counters live in parity-indexed shared cells
// so that no thread can reset a cell another thread still has to read.
#pragma once

namespace ramp {

#ifndef RAMP_CTA_F_CAP
#define RAMP_CTA_F_CAP 512     // dep-frontier records per buffer kept in shared memory (x2 buffers)
#endif
#ifndef RAMP_RQ_CAP
#define RAMP_RQ_CAP 64         // ops readied in the current tick kept in shared memory (op indices; overflow goes to HBM)
#endif
#ifndef RAMP_CTA_MIN_WARPS
#define RAMP_CTA_MIN_WARPS 16  // resident warps per SM the register allocation must allow
#endif

struct CtaCells {              // written during the tick with parity p, read after that tick's barriers, reset one tick later
    int n_ops_next;            // surviving ops copied to the next op frontier              (phase 2)
    int n_ready;               // ops readied by this tick's completions (queued op indices) (phase 2)
    int ddone, ops_done, dq_n;                                                           // (phase 2)
    int n_active;                                                                        // (phase 1)
    int arr, arr_nf, ctail;    // flow / non-flow arrival cursors, compaction cursor        (phase 3)
    unsigned long long min_op, min_dep;                                                  // (phase 1)
};

__host__ __device__ inline size_t lookahead_cta_smem(int w_cap, int c_cap, int par_cap) {
    size_t b = 0;
    b += (size_t)2 * RAMP_OPS_CAP * 16;          // op records a (ping-pong)
    b += (size_t)2 * RAMP_CTA_F_CAP * 8 * 2;     // kd, rem (two buffers)
    b += (size_t)RAMP_NF_CAP * 8;                // ready non-flow deps
    b += (size_t)2 * RAMP_OPS_CAP * 8;           // op records b
    b += (size_t)w_cap * 8;                      // done queue: {row start, degree}
    b += (size_t)RAMP_RQ_CAP * 4;                // readied-op queue
    b += (size_t)(w_cap + 2 * c_cap) * 4;        // wkey, ckey (this tick / next tick)
    b += (size_t)par_cap;                        // parent counters (bytes)
    return (b + 15) & ~(size_t)15;
}

// dep frontier entry = packed dep word (TemplateDev::dep_kd; 0 = dead entry) + remaining time
struct FrontBuf { unsigned long long* kd_sm; double* rem_sm; unsigned long long* kd_ovf; double* rem_ovf; };
__device__ __forceinline__ unsigned long long fb_kd(const FrontBuf& v, int k) { return (k < RAMP_CTA_F_CAP) ? v.kd_sm[k] : v.kd_ovf[k - RAMP_CTA_F_CAP]; }
__device__ __forceinline__ double fb_rem(const FrontBuf& v, int k) { return (k < RAMP_CTA_F_CAP) ? v.rem_sm[k] : v.rem_ovf[k - RAMP_CTA_F_CAP]; }
__device__ __forceinline__ void fb_set_kd(const FrontBuf& v, int k, unsigned long long x) { if (k < RAMP_CTA_F_CAP) v.kd_sm[k] = x; else v.kd_ovf[k - RAMP_CTA_F_CAP] = x; }
__device__ __forceinline__ void fb_set_rem(const FrontBuf& v, int k, double x) { if (k < RAMP_CTA_F_CAP) v.rem_sm[k] = x; else v.rem_ovf[k - RAMP_CTA_F_CAP] = x; }
__device__ __forceinline__ void fb_put(const FrontBuf& v, int k, unsigned long long kd, double rem) {
    if (k < RAMP_CTA_F_CAP) { v.kd_sm[k] = kd; v.rem_sm[k] = rem; }
    else { v.kd_ovf[k - RAMP_CTA_F_CAP] = kd; v.rem_ovf[k - RAMP_CTA_F_CAP] = rem; }
}

// Three block barriers per tick:
//   phase 1  op winners' min / count (B) and the min over the channel winners (D: an entry is its channel's winner iff its
//            key equals ck_cur[channel], the arg-max built during the previous tick)            -> shared cells | barrier
//   phase 2  thread 0: clock, overheads, trace (I, J).  All: H in place (survivors vote into ck_nxt, completions mark the
//            entry dead, bump the child's parent counter and append readied ops), G part 1 (op winners tick; survivors go
//            to the next op frontier, rows of completed ops to the done queue)                                  | barrier
//   phase 3  G part 2: rows of the done queue are copied to the frontier tail (arrivals vote into ck_nxt), the frontier is
//            compacted into the other buffer when more than half of it is dead, and phase A of the NEXT tick (per-worker
//            arg-max over the next op frontier) runs here too                                                   | barrier
template <int NW>
__global__ void __launch_bounds__(NW * 32, RAMP_CTA_MIN_WARPS / NW) ramp_lookahead_cta_kernel(const LookaheadArgs a) {
    constexpr int NT = NW * 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const unsigned FULL = 0xffffffffu;
    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const int warp = tid >> 5;
    const unsigned lt_mask = (1u << lane) - 1u;

    // layout by decreasing alignment
    int4* ops_a_sm0 = reinterpret_cast<int4*>(smem_raw);                                  // [2][RAMP_OPS_CAP]
    unsigned long long* kd_sm0 = reinterpret_cast<unsigned long long*>(ops_a_sm0 + 2 * RAMP_OPS_CAP);   // [2][F_CAP]
    double* rem_sm0 = reinterpret_cast<double*>(kd_sm0 + 2 * RAMP_CTA_F_CAP);            // [2][F_CAP]
    unsigned long long* nf_sm = reinterpret_cast<unsigned long long*>(rem_sm0 + 2 * RAMP_CTA_F_CAP);   // [RAMP_NF_CAP]
    int2* ops_b_sm0 = reinterpret_cast<int2*>(nf_sm + RAMP_NF_CAP);                       // [2][RAMP_OPS_CAP]
    int2* doneq = ops_b_sm0 + 2 * RAMP_OPS_CAP;                                           // [w_cap] rows of ops completed this tick
    int32_t* rq_sm = reinterpret_cast<int32_t*>(doneq + a.w_cap);                         // [RAMP_RQ_CAP]
    uint32_t* wkey = reinterpret_cast<uint32_t*>(rq_sm + RAMP_RQ_CAP);                    // [w_cap]
    uint32_t* ckey0 = wkey + a.w_cap;                                                     // [2][c_cap]
    uint32_t* par_sm = ckey0 + 2 * a.c_cap;                                               // [par_cap / 4] byte parent counters

    __shared__ CtaCells cells[2];
    __shared__ int s_work;
    __shared__ long long s_trace_off;

    unsigned char* slab = a.scratch + (uint64_t)blockIdx.x * a.scratch_stride;
    const uint64_t trace_region = a.scratch_stride - align_up((uint64_t)a.trace_cap * 12, 16);
    const double INF = __longlong_as_double(RAMP_INF_BITS);

    for (;;) {
        if (tid == 0) s_work = atomicAdd(a.cursor, 1);
        __syncthreads();
        const int wi = s_work;
        if (wi >= *a.n_work) break;
        const WorkItem item = a.items[wi];
        const TemplateDev& T = a.templates[item.template_id];
        const int N = T.n_ops, E = T.n_deps, W = T.n_workers, C = T.n_channels;
        const ScratchView sv = carve(slab, N, E, trace_region, a.trace_cap);

        const int4* __restrict__ t_op_rec = T.op_rec;
        const int2* __restrict__ t_op_row = T.op_row;
        const uint16_t* __restrict__ t_n_parents = T.op_n_parents;
        const unsigned long long* __restrict__ t_dep_kd = T.dep_kd;
        const double* __restrict__ t_dep_rt = T.dep_rt;
        uint32_t* par_done = sv.par_done;
        unsigned long long* nf_ovf = sv.nf_ovf;
        int32_t* rq_ovf = sv.rq_ovf;
        const bool psm = T.par_in_smem != 0;
        const uint32_t kmask = T.kd_kmask, cmask = T.kd_cmask;
        const int csh = T.kd_cshift, fsh = T.kd_fshift, dsh = T.kd_dshift;

        FrontBuf F, Falt;
        F.kd_sm = kd_sm0; F.rem_sm = rem_sm0; F.kd_ovf = sv.f_km_ovf; F.rem_ovf = sv.f_rem_ovf;
        Falt.kd_sm = kd_sm0 + RAMP_CTA_F_CAP; Falt.rem_sm = rem_sm0 + RAMP_CTA_F_CAP; Falt.kd_ovf = sv.f_km_ovf2; Falt.rem_ovf = sv.f_rem_ovf2;
        OpsView ops, ops_n;
        ops.a_sm = ops_a_sm0; ops.b_sm = ops_b_sm0; ops.a_ovf = sv.ops_a_ovf[0]; ops.b_ovf = sv.ops_b_ovf[0];
        ops_n.a_sm = ops_a_sm0 + RAMP_OPS_CAP; ops_n.b_sm = ops_b_sm0 + RAMP_OPS_CAP; ops_n.a_ovf = sv.ops_a_ovf[1]; ops_n.b_ovf = sv.ops_b_ovf[1];
        uint32_t* ck_cur = ckey0;
        uint32_t* ck_nxt = ckey0 + a.c_cap;

        // ---- init (JOB:432-484) ----
        if (psm) { for (int i = tid; i < (N + 3) / 4; i += NT) par_sm[i] = 0u; }
        else { for (int i = tid; i < N; i += NT) par_done[i] = 0u; }
        for (int i = tid; i < W; i += NT) wkey[i] = 0u;
        for (int i = tid; i < 2 * a.c_cap; i += NT) ckey0[i] = 0u;
        for (int k = tid; k < T.n_src; k += NT) {
            const int op = __ldg(&T.src_ops[k]);
            ops_put(ops, k, __ldg(&t_op_rec[op]), __ldg(&t_op_row[op]));          // RCE:1334
        }
        if (tid == 0) {
            for (int q = 0; q < 2; ++q) {
                cells[q].n_ops_next = 0; cells[q].n_ready = 0; cells[q].ddone = 0; cells[q].ops_done = 0; cells[q].dq_n = 0;
                cells[q].n_active = 0; cells[q].arr = 0; cells[q].arr_nf = 0; cells[q].ctail = 0;
                cells[q].min_op = RAMP_INF_BITS; cells[q].min_dep = RAMP_INF_BITS;
            }
        }
        __syncthreads();

        // CTA-uniform state (every thread holds the same values)
        int nO = T.n_src, nF = 0, live = 0, nNF = 0, ops_completed = 0, deps_completed = 0;   // nNF: ready non-flow deps (one-tick lives)
        int tick_no = 0, status = RAMP_ST_OK, par = 0;
        bool a_done = false;                         // phase A of this tick already ran during the previous tick's phase 3
        double t = 0.0, comm = 0.0, comp = 0.0;      // thread 0

        for (;;) {
            CtaCells& cc = cells[par];
            const bool big_ops = nO > 32 * NT;

            // ---- A ----
            if (!a_done) {
                for (int k = tid; k < nO; k += NT) {
                    int4 ra; int2 rb;
                    ops_get(ops, k, ra, rb);
                    atomicMax(&wkey[ra.w], (uint32_t)ra.z);
                }
                __syncthreads();
            }

            // ---- phase 1: B, C, D ----
            const bool any_nf = nNF > 0;
            uint32_t win_mask = 0u;
            {
                double mo = INF, md = INF;
                int na = 0, j = 0;
                for (int k = tid; k < nO; k += NT, ++j) {
                    int4 ra; int2 rb;
                    ops_get(ops, k, ra, rb);
                    if (wkey[ra.w] == (uint32_t)ra.z) {
                        if (j < 32) win_mask |= 1u << j;
                        ++na;
                        const double rem = __hiloint2double(ra.y, ra.x);
                        mo = (rem < mo) ? rem : mo;
                    }
                }
                if (!any_nf) {
                    for (int k = tid; k < nF; k += NT) {
                        const unsigned long long kd = fb_kd(F, k);
                        const uint32_t c = (uint32_t)(kd >> csh) & cmask;
                        if (kd != 0ull && c != cmask && ck_cur[c] == ((uint32_t)kd & kmask)) {
                            const double rem = fb_rem(F, k);
                            md = (rem < md) ? rem : md;
                        }
                    }
                }
                mo = warp_min_f64(mo);
                md = warp_min_f64(md);
                na = warp_sum_i32(na);
                if (lane == 0) {
                    const unsigned long long bo = (unsigned long long)__double_as_longlong(mo);
                    const unsigned long long bd = (unsigned long long)__double_as_longlong(md);
                    if (bo != RAMP_INF_BITS) atomicMin(&cc.min_op, bo);
                    if (bd != RAMP_INF_BITS) atomicMin(&cc.min_dep, bd);
                    if (na) atomicAdd(&cc.n_active, na);
                }
            }
            __syncthreads();

            // ---- E ----
            const double t_op = __longlong_as_double((long long)cc.min_op);
            const double t_comm = any_nf ? 0.0 : __longlong_as_double((long long)cc.min_dep);
            const double tick = (t_comm < t_op) ? t_comm : t_op;
            const int n_active = cc.n_active;

            // ---- phase 2.  I, J (thread 0) + reset of the other parity's cells (last read before this tick's first barrier) ----
            if (tid == 0) {
                const bool ticked_ops = n_active > 0;
                const bool ticked_flows = (!any_nf) && (live > 0);
                if (ticked_ops && ticked_flows) { comm = __dadd_rn(comm, tick); comp = __dadd_rn(comp, tick); }
                else if (ticked_flows) comm = __dadd_rn(comm, tick);
                else if (ticked_ops) comp = __dadd_rn(comp, tick);
                t = __dadd_rn(t, tick);
                if (tick_no < a.trace_cap) { sv.tr_n[tick_no] = n_active; sv.tr_tick[tick_no] = tick; }
                else status = RAMP_ST_TRACE_OVERFLOW;
                CtaCells& o = cells[par ^ 1];
                o.n_ops_next = 0; o.n_ready = 0; o.ddone = 0; o.ops_done = 0; o.dq_n = 0; o.n_active = 0;
                o.arr = 0; o.arr_nf = 0; o.ctail = 0;
                o.min_op = RAMP_INF_BITS; o.min_dep = RAMP_INF_BITS;
            }
            ++tick_no;
            // a tick that freezes the flows (any_nf) leaves the winners table as it is: its arrivals vote into ck_cur
            if (!any_nf) { for (int c = tid; c < C; c += NT) ck_cur[c] = 0u; }   // else: this table is the next tick's "next"
            uint32_t* ck_vote = any_nf ? ck_cur : ck_nxt;

            // ---- H.  A tick with ready non-flow deps is a zero-length tick that completes exactly those (RCE:412-422, 718-731)
            //      and leaves the flows untouched.  Any other tick ticks every flow of the pre-tick snapshot [0, nF): groups of
            //      32 entries dealt round-robin to the warps (last warps first; warp 0 also holds thread 0), in place:
            //      completed entries are marked dead ----
            if (any_nf) {
                const int n_groups = (nNF + 31) / 32;
                for (int gi = NW - 1 - warp; gi < n_groups; gi += NW) {
                    const int k = gi * 32 + lane;
                    const bool valid = k < nNF;
                    uint32_t cnt = 0u, np = 1u;
                    int child = 0;
                    if (valid) {                                                                     // JOB:525-536
                        const unsigned long long kd = (k < RAMP_NF_CAP) ? nf_sm[k] : nf_ovf[k - RAMP_NF_CAP];
                        child = (int)(kd >> dsh);
                        cnt = par_inc(psm, par_sm, par_done, child);                                 // JOB:530
                        np = psm ? (uint32_t)(kd >> (fsh + 1)) & 0xFFu : (uint32_t)__ldg(&t_n_parents[child]);
                    }
                    const bool readied = valid && (cnt == np);                                        // JOB:531 (fires once)
                    const unsigned m = __ballot_sync(FULL, readied);
                    if (m) {                         // queue the op index; its record is fetched in phase 3, all of a tick in one batch
                        const int leader = __ffs(m) - 1;
                        int base = 0;
                        if (lane == leader) base = atomicAdd(&cc.n_ready, __popc(m));
                        base = __shfl_sync(FULL, base, leader);
                        if (readied) { const int q = base + __popc(m & lt_mask); if (q < RAMP_RQ_CAP) rq_sm[q] = child; else rq_ovf[q - RAMP_RQ_CAP] = child; }
                    }
                }
            } else {
                int ddone = 0;
                const int n_groups = (nF + 31) / 32;
                // one group of 32 entries; INSM: the group lies in the shared-memory part of the frontier
                auto h_group = [&](auto insm_tag, const int gi) {
                    constexpr bool INSM = decltype(insm_tag)::value;
                    const int k = gi * 32 + lane;
                    unsigned long long kd = 0ull;
                    if (k < nF) kd = INSM ? F.kd_sm[k] : fb_kd(F, k);
                    const bool alive = kd != 0ull;
                    double r2 = 1.0;
                    if (alive) r2 = tick_down(INSM ? F.rem_sm[k] : fb_rem(F, k), tick);              // JOB:561
                    const bool done = alive && (r2 == 0.0);                                          // JOB:562
                    const uint32_t c = (uint32_t)(kd >> csh) & cmask;
                    if (alive && !done) {
                        if (INSM) F.rem_sm[k] = r2; else fb_set_rem(F, k, r2);
                        if (c != cmask) atomicMax(&ck_nxt[c], (uint32_t)kd & kmask);                 // RCE:665-689 for the next tick
                    }
                    const unsigned dmask = __ballot_sync(FULL, done);
                    if (dmask != 0u) {                                                               // JOB:525-536
                        uint32_t cnt = 0u, np = 1u;
                        int child = 0;
                        if (done) {
                            child = (int)(kd >> dsh);
                            if (INSM) F.kd_sm[k] = 0ull; else fb_set_kd(F, k, 0ull);
                            cnt = par_inc(psm, par_sm, par_done, child);                             // JOB:530
                            np = psm ? (uint32_t)(kd >> (fsh + 1)) & 0xFFu : (uint32_t)__ldg(&t_n_parents[child]);
                        }
                        ddone += __popc(dmask);
                        const bool readied = done && (cnt == np);                                     // JOB:531 (fires once)
                        const unsigned m = __ballot_sync(FULL, readied);
                        if (m) {                     // queue the op index; its record is fetched in phase 3
                            const int leader = __ffs(m) - 1;
                            int base = 0;
                            if (lane == leader) base = atomicAdd(&cc.n_ready, __popc(m));
                            base = __shfl_sync(FULL, base, leader);
                            if (readied) { const int q = base + __popc(m & lt_mask); if (q < RAMP_RQ_CAP) rq_sm[q] = child; else rq_ovf[q - RAMP_RQ_CAP] = child; }
                        }
                    }
                };
                for (int gi = NW - 1 - warp; gi < n_groups; gi += NW) {
                    if (gi * 32 + 32 <= RAMP_CTA_F_CAP) h_group(std::true_type{}, gi);
                    else h_group(std::false_type{}, gi);
                }
                if (lane == 0 && ddone) atomicAdd(&cc.ddone, ddone);
            }
            // ---- G part 1: tick the op winners (RCE:691-716); rows of completed ops are queued for the cooperative copy below ----
            {
                int j = 0, done_local = 0;
                for (int kb = 0; kb < nO; kb += NT, ++j) {
                    const int k = kb + tid;
                    const bool valid = k < nO;
                    int4 ra = make_int4(0, 0, 0, 0);
                    int2 rb = make_int2(0, 0);
                    bool done = false;
                    if (valid) {
                        ops_get(ops, k, ra, rb);
                        bool win;
                        if (big_ops) win = wkey[ra.w] == (uint32_t)ra.z;
                        else { win = ((win_mask >> j) & 1u) != 0u; if (win) wkey[ra.w] = 0u; }   // release the winner slot
                        if (win) {
                            const double rem = tick_down(__hiloint2double(ra.y, ra.x), tick);   // JOB:555
                            if (rem == 0.0) done = true;                                        // JOB:556
                            else { ra.x = __double2loint(rem); ra.y = __double2hiint(rem); }
                        }
                    }
                    const bool keep = valid && !done;
                    const unsigned mk = __ballot_sync(FULL, keep);
                    if (mk) {
                        const int leader = __ffs(mk) - 1;
                        int base = 0;
                        if (lane == leader) base = atomicAdd(&cc.n_ops_next, __popc(mk));
                        base = __shfl_sync(FULL, base, leader);
                        if (keep) ops_put(ops_n, base + __popc(mk & lt_mask), ra, rb);
                    }
                    const unsigned dm = __ballot_sync(FULL, done);
                    if (dm) {
                        const int leader = __ffs(dm) - 1;
                        int base = 0;
                        if (lane == leader) base = atomicAdd(&cc.dq_n, __popc(dm));
                        base = __shfl_sync(FULL, base, leader);
                        if (done) doneq[base + __popc(dm & lt_mask)] = rb;      // <= 1 completed op per worker per tick
                        done_local += __popc(dm);
                    }
                }
                if (lane == 0 && done_local) atomicAdd(&cc.ops_done, done_local);
            }
            __syncthreads();

            // ---- phase 3 ----
            const int nq = cc.dq_n;
            const int ddone_all = cc.ddone;                      // flows completed by this tick (0 in a zero-length tick)
            const int n_kept = cc.n_ops_next, n_ready = cc.n_ready;
            const int nO_next = n_kept + n_ready;                // next op frontier = surviving ops, then the readied ones
            const int live_after = live - ddone_all;
            // compaction when more than half of the frontier is dead (order is irrelevant: arg-max is by key)
            const bool compact = !any_nf && nF > 2 * live_after + NT;
            const FrontBuf& Fdst = compact ? Falt : F;
            const int base_off = compact ? live_after : nF;          // arrivals go behind the survivors

            // records of the readied ops: one load per thread issued now, stored at the end of the phase (the loads fly while
            // the rows are copied)
            int4 rdy_a = make_int4(0, 0, 0, 0);
            int2 rdy_b = make_int2(0, 0);
            if (tid < n_ready) {
                const int child = (tid < RAMP_RQ_CAP) ? rq_sm[tid] : rq_ovf[tid - RAMP_RQ_CAP];
                rdy_a = __ldg(&t_op_rec[child]);
                rdy_b = __ldg(&t_op_row[child]);
            }

            // G part 2: JOB:496-506 out-edges of the completed ops become ready: each warp takes every NW-th queued row and
            // copies its rows as one flattened range (all template loads of a batch in flight together)
            if (nq > 0) {
                for (int qb = 0; qb < nq; qb += 32 * NW) {
                    const int q = qb + lane * NW + warp;
                    int2 row = make_int2(0, 0);
                    if (q < nq) row = doneq[q];
                    int inc = row.y;
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const int v = __shfl_up_sync(FULL, inc, o);
                        if (lane >= o) inc += v;
                    }
                    const int total = __shfl_sync(FULL, inc, 31);
                    const int exc = inc - row.y;
                    for (int jb = 0; jb < total; jb += 32 * RAMP_U) {
                        unsigned long long kd[RAMP_U];
                        double rt[RAMP_U];
#pragma unroll
                        for (int u = 0; u < RAMP_U; ++u) {
                            kd[u] = 0ull; rt[u] = 0.0;
                            if (jb + u * 32 >= total) continue;              // warp-uniform: nothing left for this slice
                            const int jf = jb + u * 32 + lane;
                            const int jc = jf < total ? jf : total - 1;
                            int lo = 0;
#pragma unroll
                            for (int step = 16; step > 0; step >>= 1) {
                                const int v = __shfl_sync(FULL, inc, lo + step - 1);
                                if (v <= jc) lo += step;
                            }
                            const int o_start = __shfl_sync(FULL, row.x, lo);
                            const int o_exc = __shfl_sync(FULL, exc, lo);
                            const int e = o_start + (jc - o_exc);
                            if (jf < total) {
                                kd[u] = __ldg(&t_dep_kd[e]);
                                rt[u] = __ldg(&t_dep_rt[e]);                                    // RCE:542-560
                            }
                        }
#pragma unroll
                        for (int u = 0; u < RAMP_U; ++u) {
                            if (jb + u * 32 >= total) continue;              // warp-uniform
                            const int jf = jb + u * 32 + lane;
                            const bool valid = jf < total;
                            const bool flow = valid && (((kd[u] >> fsh) & 1ull) != 0ull);
                            const unsigned fm = __ballot_sync(FULL, flow);
                            const unsigned nm = __ballot_sync(FULL, valid && !flow);
                            int fbase = 0, nbase = 0;
                            if (lane == 0) {
                                if (fm) fbase = atomicAdd(&cc.arr, __popc(fm));
                                if (nm) nbase = atomicAdd(&cc.arr_nf, __popc(nm));
                            }
                            fbase = base_off + __shfl_sync(FULL, fbase, 0);
                            nbase = __shfl_sync(FULL, nbase, 0);
                            if (flow) {
                                fb_put(Fdst, fbase + __popc(fm & lt_mask), kd[u], rt[u]);
                                const uint32_t c = (uint32_t)(kd[u] >> csh) & cmask;
                                if (c != cmask) atomicMax(&ck_vote[c], (uint32_t)kd[u] & kmask);
                            } else if (valid) {
                                const int q = nbase + __popc(nm & lt_mask);
                                if (q < RAMP_NF_CAP) nf_sm[q] = kd[u]; else nf_ovf[q - RAMP_NF_CAP] = kd[u];
                            }
                        }
                    }
                }
            }
            if (compact) {
                for (int kb = 0; kb < nF; kb += NT) {
                    const int k = kb + tid;
                    unsigned long long w = 0ull;
                    if (k < nF) w = fb_kd(F, k);
                    const bool keep = w != 0ull;
                    const unsigned m = __ballot_sync(FULL, keep);
                    if (m) {
                        const int leader = __ffs(m) - 1;
                        int base = 0;
                        if (lane == leader) base = atomicAdd(&cc.ctail, __popc(m));
                        base = __shfl_sync(FULL, base, leader);
                        if (keep) fb_put(Falt, base + __popc(m & lt_mask), w, fb_rem(F, k));
                    }
                }
            }
            // phase A of the next tick: every winner slot was released in G part 1 (all of wkey is zero again)
            const bool a_next = !big_ops && (nO_next <= 32 * NT);
            if (a_next) {
                for (int k = tid; k < n_kept; k += NT) {
                    int4 ra; int2 rb;
                    ops_get(ops_n, k, ra, rb);
                    atomicMax(&wkey[ra.w], (uint32_t)ra.z);
                }
            } else if (big_ops) {
                for (int i = tid; i < W; i += NT) wkey[i] = 0u;
            }
            if (tid < n_ready) {
                ops_put(ops_n, n_kept + tid, rdy_a, rdy_b);
                if (a_next) atomicMax(&wkey[rdy_a.w], (uint32_t)rdy_a.z);
            }
            for (int k = NT + tid; k < n_ready; k += NT) {
                const int child = (k < RAMP_RQ_CAP) ? rq_sm[k] : rq_ovf[k - RAMP_RQ_CAP];
                const int4 ra = __ldg(&t_op_rec[child]);
                ops_put(ops_n, n_kept + k, ra, __ldg(&t_op_row[child]));
                if (a_next) atomicMax(&wkey[ra.w], (uint32_t)ra.z);
            }
            __syncthreads();

            // ---- K, L + frontier bookkeeping: every thread derives the same values from the shared cells ----
            const int arrived = cc.arr;
            deps_completed += ddone_all + (any_nf ? nNF : 0);
            ops_completed += cc.ops_done;
            live = live_after + arrived;
            nNF = cc.arr_nf;                                  // the previous non-flow deps were all consumed by this tick
            const bool finished = (ops_completed == N) && (deps_completed == E);     // JOB:549-551
            if (!finished && isinf(tick) && tid == 0) status = RAMP_ST_INFINITE_TICK; // RCE:462
            if (finished || isinf(tick)) break;
            if (compact) { const FrontBuf tmp = F; F = Falt; Falt = tmp; }
            nF = base_off + arrived;
            nO = nO_next;
            a_done = a_next;
            { const OpsView tmp = ops; ops = ops_n; ops_n = tmp; }
            if (!any_nf) { uint32_t* tmp = ck_cur; ck_cur = ck_nxt; ck_nxt = tmp; }
            par ^= 1;
        }
        __syncthreads();

        // ---- results (RCE:450-452) ----
        const int n_rec = tick_no < a.trace_cap ? tick_no : a.trace_cap;
        __shared__ double s_jct;
        __shared__ int s_can_util;
        const double steps = (double)T.num_training_steps;
        const int nmw = item.n_mounted_workers > 0 ? item.n_mounted_workers : W;
        double* term = sv.f_rem_ovf2;                 // the (now free) head of the dep-frontier overflow area
        if (tid == 0) {
            s_jct = __dmul_rn(t, steps);
            s_can_util = (status == RAMP_ST_OK) && (tick_no <= a.trace_cap) && (n_rec <= E);
        }
        __syncthreads();
        if (s_can_util) util_terms(sv.tr_n, sv.tr_tick, term, n_rec, (double)nmw, s_jct, tid, NT);
        __syncthreads();
        if (tid == 0) {
            a.res.jct[item.slot] = s_jct;
            a.res.comm[item.slot] = __dmul_rn(comm, steps);
            a.res.comp[item.slot] = __dmul_rn(comp, steps);
            a.res.n_ticks[item.slot] = tick_no;
            a.res.util[item.slot] = s_can_util ? util_sum(term, n_rec) : 0.0;
            a.res.util_nmw[item.slot] = s_can_util ? nmw : -1;
            long long off = -1;
            if (a.pool.top != nullptr) {
                const unsigned long long o = atomicAdd(a.pool.top, (unsigned long long)n_rec);
                if (o + (unsigned long long)n_rec <= a.pool.len) off = (long long)o;
                else if (status == RAMP_ST_OK) status = RAMP_ST_TRACE_OVERFLOW;
            }
            a.res.trace_off[item.slot] = off;
            a.res.status[item.slot] = status;
            s_trace_off = off;
            if (a.stats) {
                atomicAdd(&a.stats->lookaheads, 1ull);
                atomicAdd(&a.stats->alg_bytes, (unsigned long long)(T.algorithmic_bytes_static + 12ull * (unsigned long long)tick_no));
            }
        }
        __syncthreads();
        if (s_trace_off >= 0) {
            for (int k = tid; k < n_rec; k += NT) {
                a.pool.n_active[s_trace_off + k] = sv.tr_n[k];
                a.pool.tick[s_trace_off + k] = sv.tr_tick[k];
            }
        }
        __syncthreads();
    }
}

}  // namespace ramp
