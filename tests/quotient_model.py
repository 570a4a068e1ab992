"""Pure-Python twin of the symmetry quotient the engine applies at template registration
(ddls_b200/csrc/ramp_quotient.cpp) and of the tick loop on a quotient template.

Why it is exact.  All n sub-ops of a partitioned op have the same cost, the same parents and sit on n different
servers, so in ``_run_lookahead`` (RCE:379-467) they become ready, tick and complete in the same ticks; so do the
n(n-1) flows of one original edge.  Colour refinement (1-WL) over ops and deps finds the coarsest partition in
which every member of a class sees the same things: cost / run time / flow flag, the classes of its in- and
out-deps (with multiplicity) and, for ops, its position in the priority order of its worker next to the same
classes.  A dep's state does not depend on its channel or priority (every ready flow ticks every tick,
RCE:733-775); those only feed t_comm = min over channels of remaining(winner), which is evaluated per GROUP of
channels that carry the same classes in the same priority order ("twins" -- deps leaving one op class with one run
time -- counted once).  Members of a class are therefore in the same state at every tick, and the lookahead can be
run on one representative per class, with
  * op weight    = class size (the members sit on distinct workers: each one is its worker's winner when the class
                   wins, so the trace's active-worker count adds the class size, RCE:709-715);
  * op threshold = n_parents x class size, dep inc = members of the entry: the class counter is the sum of its
                   members' ``len(parent_deps_completed)`` (JOB:530); all entries of a dep class complete in one
                   tick, and the class is readied in the tick its counter passes through the threshold -- the tick in
                   which every member's own count passes through n_parents (the ``==`` of JOB:531 fires once).
Everything else -- rank keys, winners per worker / channel group, min remaining, zero-length ticks, f64
accumulation order -- is the same algorithm on fewer items.
"""
import math
import numpy as np

from kernel_model import rank_keys


def _relabel(sigs):
    ids = {}
    out = np.empty(len(sigs), dtype=np.int64)
    for i, s in enumerate(sigs):
        out[i] = ids.setdefault(s, len(ids))
    return out, len(ids)


def quotient(job, max_rounds=256):
    """Python twin of ramp_quotient_template (exact tuples instead of hashes).  Returns ddls_b200.quotient.QuotientJob."""
    from ddls_b200.quotient import QuotientJob
    N, E, W, C = job.n_ops, job.n_deps, job.n_workers, job.n_channels
    row = job.row_ptr.astype(np.int64)
    src = np.repeat(np.arange(N, dtype=np.int64), np.diff(row))
    dst = job.dep_dst.astype(np.int64)
    op_key = np.array(rank_keys(job.op_prio), dtype=np.int64)
    dep_key = np.array(rank_keys(job.dep_prio), dtype=np.int64)
    chan = job.dep_channel.astype(np.int64)
    has_ch = (chan != 0xFFFF)
    in_deps = [[] for _ in range(N)]
    for e in range(E):
        in_deps[int(dst[e])].append(e)
    by_worker = [[] for _ in range(W)]
    for i in np.argsort(-op_key, kind='stable'):
        by_worker[int(job.op_worker[i])].append(int(i))
    wpos = np.zeros(N, dtype=np.int64)
    for ops in by_worker:
        for p, i in enumerate(ops):
            wpos[i] = p

    oc, n_oc = _relabel([(float(job.op_cost[i] + 0.0).hex(), int(job.op_n_parents[i])) for i in range(N)])
    dc, n_dc = _relabel([(float(job.dep_run_time[e] + 0.0).hex(), bool(job.dep_is_flow[e])) for e in range(E)])
    for _ in range(max_rounds):
        wsig = [tuple(oc[i] for i in ops) for ops in by_worker]
        dc2, n_dc2 = _relabel([(dc[e], oc[src[e]], oc[dst[e]]) for e in range(E)])
        oc2, n_oc2 = _relabel([(oc[i], wsig[int(job.op_worker[i])], wpos[i],
                                tuple(sorted(dc2[row[i]:row[i + 1]].tolist())),
                                tuple(sorted(int(dc2[e]) for e in in_deps[i]))) for i in range(N)])
        stable = (n_dc2 == n_dc) and (n_oc2 == n_oc)
        oc, dc, n_oc, n_dc = oc2, dc2, n_oc2, n_dc2
        if stable:
            break
    else:
        raise Exception('colour refinement did not converge')
    rep_op = np.array([np.nonzero(oc == c)[0][0] for c in range(n_oc)])
    size_op = np.bincount(oc, minlength=n_oc)

    # worker groups
    wseq = [tuple(oc[i] for i in ops) for ops in by_worker]
    wg, n_wg = _relabel(wseq)
    q_op_key = np.zeros(n_oc, dtype=np.int64)
    q_op_worker = np.zeros(n_oc, dtype=np.int64)
    seen = set()
    for w in range(W):
        g = int(wg[w])
        if g in seen:
            continue
        seen.add(g)
        for i in by_worker[w]:
            q_op_key[oc[i]] = op_key[i]
            q_op_worker[oc[i]] = g

    # twins and channel groups
    twin, _ = _relabel([(int(oc[src[e]]), float(job.dep_run_time[e] + 0.0).hex(), bool(job.dep_is_flow[e])) for e in range(E)])
    on_chan = [[] for _ in range(C)]
    for e in range(E):
        if has_ch[e]:
            on_chan[int(chan[e])].append(e)
    cseq, ckeys = [], []
    for c in range(C):
        best = {}
        for e in on_chan[c]:
            best[int(twin[e])] = max(best.get(int(twin[e]), 0), int(dep_key[e]))
        order = sorted(best.items(), key=lambda kv: -kv[1])
        cseq.append(tuple(k for k, _ in order))
        ckeys.append(dict(order))
    cg, n_cg = _relabel(cseq)
    g_keys = {}
    for c in range(C):
        g_keys.setdefault(int(cg[c]), ckeys[c])

    # one key per twin for all groups?  (see ramp_quotient.cpp)
    gk = {}
    for e in range(E):
        if has_ch[e]:
            gk[int(twin[e])] = max(gk.get(int(twin[e]), 0), int(dep_key[e]))
    seq_of_group = {}
    for c in range(C):
        seq_of_group.setdefault(int(cg[c]), cseq[c])
    merged = n_cg <= 64 and all(gk[sq[k - 1]] > gk[sq[k]] for sq in seq_of_group.values() for k in range(1, len(sq)))
    merged = merged and len(set(gk.values())) == len(gk)
    masks_valid = n_cg <= 64

    # entries
    ids, ent_rep, ent_inc, ent_mask = {}, [], [], []
    entry = np.zeros(E, dtype=np.int64)
    for e in range(E):
        g = int(cg[int(chan[e])]) if has_ch[e] else -1
        k = (int(dc[e]), (0 if g < 0 else 1) if merged else g + 1)
        if k not in ids:
            ids[k] = len(ent_rep)
            ent_rep.append(e)
            ent_inc.append(0)
            ent_mask.append(0)
        entry[e] = ids[k]
        ent_inc[ids[k]] += 1
        if g >= 0 and masks_valid:
            ent_mask[ids[k]] |= (1 << g)
    n_ent = len(ent_rep)
    order = sorted(range(n_ent), key=lambda a: int(oc[src[ent_rep[a]]]))     # stable
    new_id = np.zeros(n_ent, dtype=np.int64)
    for k, a in enumerate(order):
        new_id[a] = k
    q_row = np.zeros(n_oc + 1, dtype=np.int64)
    q_dst = np.zeros(n_ent, dtype=np.int64)
    q_rt = np.zeros(n_ent, dtype=np.float64)
    q_key = np.zeros(n_ent, dtype=np.int64)
    q_ch = np.full(n_ent, 0xFFFFFFFF, dtype=np.int64)
    q_mask = np.zeros(n_ent, dtype=np.uint64)
    q_flow = np.zeros(n_ent, dtype=np.uint8)
    q_inc = np.zeros(n_ent, dtype=np.int64)
    for k, a in enumerate(order):
        e = ent_rep[a]
        q_row[oc[src[e]] + 1] += 1
        q_dst[k] = oc[dst[e]]
        q_rt[k] = job.dep_run_time[e] + 0.0
        q_flow[k] = 1 if job.dep_is_flow[e] else 0
        q_inc[k] = ent_inc[a]
        q_mask[k] = ent_mask[a]
        if not has_ch[e]:
            q_key[k] = dep_key[e]
        elif merged:
            q_key[k] = gk[int(twin[e])]
        else:
            g = int(cg[int(chan[e])])
            q_ch[k] = g
            q_key[k] = g_keys[g][int(twin[e])]
    np.cumsum(q_row, out=q_row)
    return QuotientJob(n_ops=n_oc, n_deps=n_ent, n_workers=n_wg, n_channels=n_cg,
                       num_training_steps=job.num_training_steps,
                       op_cost=(job.op_cost[rep_op] + 0.0), op_key=q_op_key, op_worker=q_op_worker,
                       op_weight=size_op.astype(np.int64),
                       op_threshold=job.op_n_parents[rep_op].astype(np.int64) * size_op,
                       row_ptr=q_row, dep_dst=q_dst, dep_run_time=q_rt, dep_key=q_key, dep_channel=q_ch,
                       dep_is_flow=q_flow, dep_inc=q_inc, op_class=oc.astype(np.int64), dep_entry=new_id[entry],
                       dep_group_mask=q_mask, merged=int(merged), masks_valid=int(masks_valid))


def run_lookahead_quotient(q):
    """The kernels' tick loop (tests/kernel_model.py) on a quotient job: weights in the active-worker count,
    entry sizes in the (scaled) parent counters."""
    N, E = q.n_ops, q.n_deps
    row = q.row_ptr
    in_deg = np.zeros(N, dtype=np.int64)
    for e in range(E):
        in_deg[int(q.dep_dst[e])] += 1
    par_done = [0] * N
    ops = [(i, float(q.op_cost[i]) + 0.0) for i in range(N) if in_deg[i] == 0]
    flows, nf = [], []

    def groups_of(e):                       # set of channel groups of an entry as a Python int bit mask
        if q.masks_valid:
            return int(q.dep_group_mask[e])
        c = int(q.dep_channel[e])
        return 0 if c == 0xFFFFFFFF else (1 << c)
    t = comm = comp = 0.0
    trace_n, trace_tick = [], []
    ops_completed = deps_completed = 0
    INF = math.inf
    finished = False
    # the frontier peaks the thread kernel records in TemplateHints: ready op classes counted with the classes readied in the
    # tick (the kernel appends them behind the frontier before it compacts it), ready flow / non-flow entries after the tick
    max_o, max_f, max_nf = len(ops), 0, 0
    while True:
        wkey = {}
        for op, rem in ops:
            w = int(q.op_worker[op])
            wkey[w] = max(wkey.get(w, 0), int(q.op_key[op]))
        winners = [(op, rem) for op, rem in ops if wkey[int(q.op_worker[op])] == int(q.op_key[op])]
        t_op = min([rem for _, rem in winners], default=INF)
        n_active = sum(int(q.op_weight[op]) for op, _ in winners)
        any_nf = len(nf) > 0
        if any_nf:
            t_comm = 0.0
        else:
            # an entry wins on a channel group of its set unless a ready entry with a larger key lies on that group too
            t_comm = INF
            for e, rem in flows:
                open_groups = groups_of(e)
                for e2, _ in flows:
                    if int(q.dep_key[e2]) > int(q.dep_key[e]):
                        open_groups &= ~groups_of(e2)
                if open_groups and rem < t_comm:
                    t_comm = rem
        tick = t_comm if t_comm < t_op else t_op
        ticked_ops, ticked_flows = len(winners) > 0, (not any_nf) and len(flows) > 0
        if ticked_flows:
            comm += tick
        if ticked_ops:
            comp += tick
        t += tick
        trace_n.append(n_active)
        trace_tick.append(tick)
        ops_next = []

        def complete_dep(e):
            child = int(q.dep_dst[e])
            old = par_done[child]
            par_done[child] = old + int(q.dep_inc[e])
            if old < int(q.op_threshold[child]) <= par_done[child]:
                ops_next.append((child, float(q.op_cost[child]) + 0.0))
        if any_nf:
            for e in nf:
                complete_dep(e)
            deps_completed += len(nf)
            nf = []
            survivors = flows
        else:
            survivors = []
            for e, rem in flows:
                r2 = rem - (rem if rem < tick else tick)
                if r2 == 0.0:
                    complete_dep(e)
                    deps_completed += 1
                else:
                    survivors.append([e, r2])
        max_o = max(max_o, len(ops) + len(ops_next))
        win_set = {op for op, _ in winners}
        arrivals = []
        for op, rem in ops:
            if op in win_set:
                r2 = rem - (rem if rem < tick else tick)
                if r2 == 0.0:
                    ops_completed += 1
                    arrivals.extend(range(int(row[op]), int(row[op + 1])))
                    continue
                rem = r2
            ops_next.append((op, rem))
        for e in arrivals:
            if int(q.dep_is_flow[e]):
                survivors.append([e, float(q.dep_run_time[e]) + 0.0])
            else:
                nf.append(e)
        flows = survivors
        ops = ops_next
        max_f, max_nf = max(max_f, len(flows)), max(max_nf, len(nf))
        finished = ops_completed == N and deps_completed == E
        if finished or math.isinf(tick):
            break
    steps = float(q.num_training_steps)
    return dict(jct=t * steps, comm=comm * steps, comp=comp * steps, n_ticks=len(trace_tick),
                trace_n_active=np.array(trace_n, dtype=np.int32), trace_tick=np.array(trace_tick, dtype=np.float64),
                finished=finished, max_o=max_o, max_f=max_f, max_nf=max_nf)


def identity_quotient(job):
    """Every op its own class (ramp_engine.cu identity_quotient): what RAMP_LOOKAHEAD_MODE=thread_unfolded simulates."""
    from ddls_b200.quotient import QuotientJob
    job.canonicalise()
    N, E, C = job.n_ops, job.n_deps, job.n_channels
    chan = job.dep_channel.astype(np.int64)
    has_ch = chan != 0xFFFF
    masks_valid = C <= 64
    mask = np.array([(1 << int(c)) if (h and masks_valid) else 0 for c, h in zip(chan, has_ch)], dtype=np.uint64)
    return QuotientJob(n_ops=N, n_deps=E, n_workers=job.n_workers, n_channels=C, num_training_steps=job.num_training_steps,
                       op_cost=job.op_cost + 0.0, op_key=np.array(rank_keys(job.op_prio), dtype=np.int64),
                       op_worker=job.op_worker.astype(np.int64), op_weight=np.ones(N, dtype=np.int64),
                       op_threshold=job.op_n_parents.astype(np.int64), row_ptr=job.row_ptr.astype(np.int64),
                       dep_dst=job.dep_dst.astype(np.int64), dep_run_time=job.dep_run_time + 0.0,
                       dep_key=np.array(rank_keys(job.dep_prio), dtype=np.int64),
                       dep_channel=np.where(has_ch, chan, 0xFFFFFFFF), dep_is_flow=job.dep_is_flow.astype(np.uint8),
                       dep_inc=np.ones(E, dtype=np.int64), op_class=np.arange(N, dtype=np.int64),
                       dep_entry=np.arange(E, dtype=np.int64), dep_group_mask=mask, merged=0, masks_valid=int(masks_valid))
