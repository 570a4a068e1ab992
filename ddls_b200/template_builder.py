"""Synthetic Action generator: ForwardGraph + partition degree + a worker block -> LoweredJob.

The reference's job ingest (``ddls.demands.jobs``) and heuristic agents (``ramp_cluster/agents``) stay
as they are and are NOT restated here.  This module exists because neither the reference nor its
job-graph profiles exist on the GPU box: ``bench.py`` and the large ``-m gpu`` parity tests need
hot-path inputs of BASELINE.json's sizes (ResNet-50-like job, degree 16: N ~ 5.6 k ops, E ~ 140 k deps)
generated from nothing.  It follows the *shape* the reference's pipeline produces:

  * mirrored forward/backward graph, backward id = 2n-(i-1), join edge n -> n+1, edge size =
    memory cost of the source op                      (ddls/utils.py:342-415, partitioners/utils.py:36-38)
  * per forward op, an even number of splits
    ``max(1, min(ceil(ceil(cost/quantum)/2)*2, degree))``                   (RJPE:332-343)
  * op split into n sub-ops 'ida'..: cost/n, memory/n, every in/out edge fanned out to all sub-ops,
    n(n-1) bidirectional weight-sync edges between the sub-ops of a backward op  (partitioners/utils.py:42-110)

and then applies a *simple, documented* stand-in for the agents: sub-op k of every split op goes to the
k-th worker of one aligned block of ``degree`` workers (unsplit ops to worker 0 of the block); a flow's
run time is latency + 2 IO + size/bandwidth (the reference's one-to-one formula, actions/utils.py:90-99);
each flow is mounted on the single 1-hop channel (src server -> dst server); SRPT priorities (shortest
remaining time = highest priority; srpt_op_scheduler.py:16-88, srpt_dep_scheduler.py:14-83).
The hot path does not care which agent produced its inputs; parity on these templates is checked against
the CPU oracle, parity on the reference's own agents against tests/golden.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import numpy as np

from .lowered import LoweredJob, MountScalars, NO_CHANNEL
from .observation import job_arrays
from .synth import ForwardGraph


class RampShape:
    """c x r x s RAMP topology; worker index = c*(R*S) + r*S + s (ramp.py:36-41 node order, RCE:169-198)."""

    def __init__(self, c, r, s, total_node_bandwidth=1.6e12, latency=50e-9, io_latency=100e-9):
        if r > c:
            raise Exception(f'num_racks_per_communication_group ({r}) must be <= num_communication_groups ({c})')  # ramp.py:22-23
        self.c, self.r, self.s = c, r, s
        self.n_workers = c * r * s
        self.channel_bandwidth = total_node_bandwidth / c          # ramp.py:27
        self.latency, self.io_latency = latency, io_latency

    def worker_id(self, idx):
        c, rem = divmod(idx, self.r * self.s)
        r, s = divmod(rem, self.s)
        return f'node_{c}-{r}-{s}_worker_0'                       # RCE:191

    def one_to_one_time(self, size):
        return self.latency + 2 * self.io_latency + size / self.channel_bandwidth   # actions/utils.py:90-99


def _sub_id(op, k):
    return f'{op}{chr(97 + k)}'                                   # partitioners/utils.py:76


def partition_graph(fwd: ForwardGraph, degree: int, quantum: float, with_adjacency: bool = False):
    """Returns (nodes: {id(str): (cost, mem)}, edges: {(u, v): size}, n_splits per original op); with_adjacency adds the
    successor / predecessor lists in networkx's adjacency (insertion) order, which the reference's agents iterate in."""
    n = fwd.n
    mem = {}
    cost = {}
    for i in range(1, n + 1):
        m = fwd.act[i - 1] + fwd.par[i - 1]                       # utils.py:432 memory_cost = activation + parameter
        cost[str(i)], mem[str(i)] = fwd.fwd[i - 1], m
        cost[str(2 * n - (i - 1))], mem[str(2 * n - (i - 1))] = fwd.bwd[i - 1], m
    succ: Dict[str, List[str]] = {k: [] for k in cost}
    pred: Dict[str, List[str]] = {k: [] for k in cost}
    size: Dict[Tuple[str, str], float] = {}

    def add_edge(u, v, sz):
        if (u, v) not in size:
            succ[u].append(v)
            pred[v].append(u)
        size[(u, v)] = sz

    for (u, v) in fwd.edges:
        add_edge(str(u), str(v), mem[str(u)])
    for (u, v) in fwd.edges:
        bu, bv = str(2 * n - (v - 1)), str(2 * n - (u - 1))
        add_edge(bu, bv, mem[bu])
    add_edge(str(n), str(n + 1), mem[str(n)])

    splits = {}
    for i in range(1, n + 1):
        c = fwd.fwd[i - 1]
        k = int(max(1, min(math.ceil(math.ceil(c / quantum) / 2) * 2, degree)))   # RJPE:336
        splits[i] = k
    in_feat: Dict[Tuple[str, str], float] = {}
    out_feat: Dict[Tuple[str, str], float] = {}
    for i in range(1, n + 1):
        k = splits[i]
        if k <= 1:
            continue
        for which, node in enumerate((str(i), str(2 * n - (i - 1)))):
            ins, outs = list(pred[node]), list(succ[node])
            subs = [_sub_id(node, j) for j in range(k)]
            sub_cost, sub_mem = cost[node] / k, mem[node] / k
            # remove the node
            for p in ins:
                succ[p].remove(node)
                size.pop((p, node), None)
            for s_ in outs:
                pred[s_].remove(node)
                size.pop((node, s_), None)
            del succ[node], pred[node], cost[node], mem[node]
            for sid in subs:
                cost[sid], mem[sid] = sub_cost, sub_mem
                succ[sid], pred[sid] = [], []
            for sid in subs:
                for p in ins:
                    add_edge(p, sid, size.get((p, sid), 0.0))
                    in_feat[(p, sid)] = mem[p] / k
                for s_ in outs:
                    add_edge(sid, s_, size.get((sid, s_), 0.0))
                    out_feat[(sid, s_)] = mem[s_] / k
            if which == 1:                                        # weight-sync collective between backward sub-ops
                for a in subs:
                    for b in subs:
                        if a != b:
                            add_edge(a, b, 0.0)
                            in_feat[(a, b)] = sub_mem
    for e, sz in in_feat.items():                                 # nx.set_edge_attributes(in) then (out): out overrides
        if e in size:
            size[e] = sz
    for e, sz in out_feat.items():
        if e in size:
            size[e] = sz
    nodes = {k: (cost[k], mem[k]) for k in cost}
    if with_adjacency:
        return nodes, size, splits, succ, pred
    return nodes, size, splits


# Block of servers RampFirstFitOpPlacer picks for a job of `degree` sub-ops per op on an EMPTY 4x4x4 cluster, in sorted
# server-id order (probed from the unmodified reference, oracle/gen_golden.py runs; sub-op k goes to the k-th server)
REFERENCE_BLOCK_4x4x4 = {
    1: [(0, 0, 0)],
    2: [(0, 0, 0), (1, 0, 0)],
    4: [(0, 0, 0), (0, 1, 0), (1, 0, 0), (1, 1, 0)],
    8: [(c, r, s_) for c in range(2) for r in range(2) for s_ in range(2)],
    16: [(c, r, 0) for c in range(4) for r in range(4)],
}


def _all_reduce_time(message_size, node_ids, racks, cgs, x, data_rate, latency, io_latency, cont_racks=1):
    """calc_ramp_all_reduce_collective_communication_run_time (actions/utils.py:40-88), same numpy calls in the same order."""
    mem_frq, peak, bytes_per_comp = 2e12, 130e12, 2

    def trx(cg, d, J):                                            # effective_trx_per_comm, actions/utils.py:101-106
        if d == 1:
            return 0
        return 1 + (min(cg // J, cg // (d - 1)) - 1)

    def add_time(data_sz, devices):                               # get_parallel_add_comp_time_single, actions/utils.py:108-118
        n_op = np.ceil(np.log2(devices))
        n_bytes = (devices + 1) * bytes_per_comp
        ai = n_op / n_bytes
        total_ops = n_op * (data_sz / devices) / bytes_per_comp
        return total_ops / np.min([mem_frq * ai, peak])
    data_per_tx = data_rate / x
    sub = [cgs, min(cgs, node_ids), racks, np.ceil(node_ids / x)]
    bw = [trx(x, d, cont_racks) * data_per_tx for d in sub]
    msg = [np.ceil(message_size / sub[0])]
    for i in sub[1:]:
        msg.append(np.ceil(msg[-1] / i))
    comm, comp = 0.0, 0.0
    for step, d in enumerate(sub):
        if d > 1:
            comp += add_time(msg[step] * d, d)
            comm += latency + 2 * io_latency + msg[step] / bw[step]
    return 2 * comm + comp


def reference_dep_run_times(fwd: ForwardGraph, nodes, size, splits, succ, pred, coords_of_op, shape: RampShape):
    """update_dep_run_times (actions/utils.py:13-393) for one job: deps of a partitioned op whose parent and child servers
    coincide form an all-reduce collective, the backward sub-ops' mutual sync edges form 2-dep collectives, everything
    else is a one-to-one transfer; one-to-one times are applied last.  coords_of_op: op id -> (cg, rack, server) of its server.
    Returns {(u, v): init_run_time}."""
    n = fwd.n
    x = shape.c
    rt = {}

    def collective_time(deps):
        cgs, racks, nodes_, servers, message = set(), set(), set(), set(), 0
        for (u, v) in deps:                                       # get_collective_info, actions/utils.py:168-245
            for op in (u, v):
                c, r, s_ = coords_of_op[op]
                cgs.add(c); racks.add(r); nodes_.add(s_); servers.add((c, r, s_))
            message += size[(u, v)]
        if len(servers) == 1:
            return 0
        return _all_reduce_time(message, len(nodes_), len(racks), len(cgs), x, shape.channel_bandwidth, shape.latency,
                                shape.io_latency)
    collectives, one_to_one = [], []
    for i in range(1, n + 1):
        b = 2 * n - (i - 1)
        k = splits[i]
        if k > 1:
            fdeps, bdeps, sync, seen = [], [], [], set()
            for j in range(k):
                fs = _sub_id(str(i), j)
                fdeps.extend((fs, v) for v in succ[fs])
                bs = _sub_id(str(b), j)
                for p in pred[bs]:
                    if p in succ[bs]:                             # bidirectional sync edge
                        if (p, bs) not in seen and (bs, p) not in seen:
                            sync.append([(p, bs), (bs, p)])
                            seen.add((p, bs))
                    else:
                        bdeps.append((p, bs))
            for deps in (fdeps, bdeps):
                if sorted(coords_of_op[u] for (u, _) in deps) == sorted(coords_of_op[v] for (_, v) in deps):
                    collectives.append(deps)
                else:
                    one_to_one.extend(deps)
            collectives.extend(sync)
        else:
            one_to_one.extend((str(i), v) for v in succ[str(i)])
            one_to_one.extend((p, str(b)) for p in pred[str(b)])
    for deps in collectives:
        t = collective_time(deps)
        for d in deps:
            rt[d] = t
    for (u, v) in one_to_one:                                     # set_one_to_one_dep_run_time, actions/utils.py:146-166
        if coords_of_op[u] == coords_of_op[v] or size[(u, v)] == 0:
            rt[(u, v)] = 0
        else:
            rt[(u, v)] = shape.latency + 2 * shape.io_latency + size[(u, v)] / shape.channel_bandwidth
    return rt


def build_template(fwd: ForwardGraph, degree: int, shape: RampShape, block_start: int = 0, quantum: float = 0.01,
                   num_training_steps: int = 50, model_id: int = 0, max_acceptable_frac: float = 1.0,
                   run_times: str = 'one_to_one') -> LoweredJob:
    """Partition ``fwd`` to ``degree``, place it on workers [block_start, block_start+degree) and lower it.

    run_times='one_to_one' (default, the bench's stand-in): every flow takes the one-to-one transfer time.
    run_times='reference': the reference's update_dep_run_times (collectives) and SRPT dep priorities over ALL deps in graph
    edge order, on the block RampFirstFitOpPlacer picks on an empty 4x4x4 cluster -- reproduces the reference pipeline's
    lowered job array for array (tests/test_lowering_roundtrip.py against tests/golden/resnet64_deg*_full.npz)."""
    if degree != 1 and degree % 2 != 0:
        raise Exception(f'Invalid num_partitions={degree}; RAMP placer expects even numbers.')   # op_partition.py:26-27
    if block_start + max(degree, 1) > shape.n_workers:
        raise Exception('worker block does not fit in the cluster')
    nodes, size, splits, succ, pred = partition_graph(fwd, degree, quantum, with_adjacency=True)
    op_ids = sorted(nodes)                                        # string sort == RCE:56
    idx = {op: i for i, op in enumerate(op_ids)}
    N = len(op_ids)
    op_cost = np.array([nodes[o][0] for o in op_ids], dtype=np.float64)

    def local_worker(op):
        last = op[-1]
        return (ord(last) - 97) if last.isalpha() else 0
    op_worker_local = np.array([local_worker(o) for o in op_ids], dtype=np.int64)
    used = sorted(set(op_worker_local.tolist()))
    remap = {w: i for i, w in enumerate(used)}
    op_worker = np.array([remap[w] for w in op_worker_local], dtype=np.uint16)
    worker_ids = [shape.worker_id(block_start + w) for w in used]

    dep_ids = sorted((u, v, 0) for (u, v) in size)
    E = len(dep_ids)
    src = np.array([idx[u] for (u, _, _) in dep_ids], dtype=np.int64)
    dst = np.array([idx[v] for (_, v, _) in dep_ids], dtype=np.int32)
    sizes = np.array([size[(u, v)] for (u, v, _) in dep_ids], dtype=np.float64)
    row_ptr = np.zeros(N + 1, dtype=np.int32)
    np.add.at(row_ptr, src + 1, 1)
    np.cumsum(row_ptr, out=row_ptr)
    sw, dw = op_worker[src].astype(np.int64), op_worker[dst].astype(np.int64)
    is_flow = ((sw != dw) & (sizes != 0)).astype(np.uint8)        # RCE:531-536 (one worker per server RCE:180)
    run_time = np.where(is_flow == 1, shape.latency + 2 * shape.io_latency + sizes / shape.channel_bandwidth, 0.0)
    all_dep_order = None
    if run_times == 'reference':
        if (shape.c, shape.r, shape.s) != (4, 4, 4) or degree not in REFERENCE_BLOCK_4x4x4 or block_start != 0:
            raise Exception("run_times='reference' is available for the probed empty-cluster blocks of a 4x4x4 RAMP only")
        block = REFERENCE_BLOCK_4x4x4[degree]
        coords_of_op = {o: block[int(op_worker[idx[o]])] for o in op_ids}
        worker_ids = [f'node_{c}-{r}-{s_}_worker_0' for (c, r, s_) in block[:len(used)]]
        rt_map = reference_dep_run_times(fwd, nodes, size, splits, succ, pred, coords_of_op, shape)
        run_time = np.array([float(rt_map[(u, v)]) for (u, v, _) in dep_ids], dtype=np.float64)
        run_time = np.where(is_flow == 1, run_time, 0.0)          # RCE:542-560
        dep_index = {(u, v): e for e, (u, v, _) in enumerate(dep_ids)}
        all_dep_order = [dep_index[(u, v)] for u in nodes for v in succ[u]]    # job.computation_graph.edges order
        sched_cost = np.array([float(rt_map[(u, v)]) for (u, v, _) in dep_ids], dtype=np.float64)
    W = len(used)
    chan_key = sw * W + dw
    flow_keys = np.unique(chan_key[is_flow == 1])
    chan_index = {int(k): i for i, k in enumerate(flow_keys)}
    dep_channel = np.full(E, NO_CHANNEL, dtype=np.uint16)
    fl = np.nonzero(is_flow)[0]
    dep_channel[fl] = [chan_index[int(k)] for k in chan_key[fl]]
    channel_ids = []
    for k in flow_keys:
        a, b = divmod(int(k), W)
        na = worker_ids[a].split('node_')[1].split('_worker')[0]
        nb = worker_ids[b].split('node_')[1].split('_worker')[0]
        channel_ids.append(f'src_{na}_dst_{nb}_channel_0')       # utils.py:550-555

    # SRPT: highest cost -> priority 0, ... (ties: lower index first in the descending order)
    op_prio = np.zeros(N, dtype=np.int64)
    for w in range(W):
        members = np.nonzero(op_worker == w)[0]
        order = members[np.argsort(-op_cost[members], kind='stable')]
        op_prio[order] = np.arange(len(order))
    dep_prio = np.zeros(E, dtype=np.int64)
    if all_dep_order is not None:
        # SRPTDepScheduler (srpt_dep_scheduler.py:14-83): ALL deps in graph edge order, stable descending sort by run time
        ordered = np.array(all_dep_order, dtype=np.int64)
        ranked = ordered[np.argsort(-sched_cost[ordered], kind='stable')]
        prio_all = np.zeros(E, dtype=np.int64)
        prio_all[ranked] = np.arange(E)
        dep_prio[fl] = prio_all[fl]                               # the lowering reads priorities of placed flows only
    elif len(fl):
        order = fl[np.argsort(-run_time[fl], kind='stable')]
        dep_prio[order] = np.arange(len(order))

    # parents = predecessors that are not also successors (JOB:508-523)
    pair = set(zip(src.tolist(), dst.tolist()))
    n_parents = np.zeros(N, dtype=np.int64)
    for (a, b) in pair:
        if (b, a) not in pair:
            n_parents[b] += 1

    seq_time = float(sum(nodes[o][0] for o in nodes)) * num_training_steps     # JOB:224-235
    mount = MountScalars(max_acceptable_jct=max_acceptable_frac * seq_time,
                         part_op_mem=float(sum(nodes[o][1] for o in nodes)),
                         part_dep_size=float(sizes.sum()),
                         flow_size=float(sizes[is_flow == 1].sum()),
                         n_mounted_workers=W, n_mounted_channels=len(channel_ids))
    lj = LoweredJob(n_ops=N, n_deps=E, n_workers=W, n_channels=len(channel_ids), num_training_steps=num_training_steps,
                    model_id=model_id, degree=degree, op_cost=op_cost, op_prio=op_prio, op_worker=op_worker,
                    op_n_parents=n_parents.astype(np.uint16), row_ptr=row_ptr, dep_dst=dst, dep_run_time=run_time,
                    dep_prio=dep_prio, dep_channel=dep_channel, dep_is_flow=is_flow, mount=mount, model=fwd.name,
                    op_ids=op_ids, dep_ids=dep_ids, worker_ids=worker_ids, channel_ids=channel_ids)
    lj.seq_time = seq_time
    return lj.canonicalise()


def original_job_totals(fwd: ForwardGraph):
    """(job_total_op_memory_cost, job_total_dep_size) of the un-partitioned mirrored job (JOB:237-248): the ops' memory costs
    (activation + parameters) and the deps' sizes (the source op's activation, utils.py:394-396) summed in the job graph's node /
    edge iteration order -- ``observation.job_arrays``' totals, so the arrival rows carry the reference's values bit for bit."""
    a = job_arrays(fwd)
    return a['total_op_memory'], a['total_dep_size']


def random_dag_template(rng: np.random.Generator, n_ops: int, avg_out: float = 3.0, n_workers: int = 4,
                        p_mutual: float = 0.05, p_zero_cost: float = 0.1, p_tie: float = 0.3, p_nonflow: float = 0.3,
                        model_id: int = 0, degree: int = 2) -> LoweredJob:
    """Adversarial random lowered job for property tests: priority ties, zero-cost ops, zero-time flows,
    flows without a channel, mutual (sync) edge pairs, several sources."""
    N = n_ops
    edges = set()
    for v in range(1, N):
        k = 1 + rng.poisson(max(avg_out - 1, 0))
        for u in rng.integers(0, v, size=min(k, v)):
            edges.add((int(u), v))
    # mutual pairs between ops that share all parents (like backward sub-ops): pick siblings
    sib = list(range(N))
    rng.shuffle(sib)
    for a, b in zip(sib[::2], sib[1::2]):
        if rng.random() < p_mutual and (a, b) not in edges and (b, a) not in edges:
            edges.add((a, b)); edges.add((b, a))
    dep_ids = sorted(edges)
    E = len(dep_ids)
    src = np.array([u for u, _ in dep_ids], dtype=np.int64)
    dst = np.array([v for _, v in dep_ids], dtype=np.int32)
    row_ptr = np.zeros(N + 1, dtype=np.int32)
    np.add.at(row_ptr, src + 1, 1)
    np.cumsum(row_ptr, out=row_ptr)
    pair = set(dep_ids)
    n_parents = np.zeros(N, dtype=np.int64)
    for (a, b) in pair:
        if (b, a) not in pair:
            n_parents[b] += 1
    op_cost = np.round(rng.uniform(0.05, 2.0, size=N), 3)
    op_cost[rng.random(N) < p_zero_cost] = 0.0
    op_worker = rng.integers(0, n_workers, size=N).astype(np.uint16)
    op_worker[:n_workers] = np.arange(n_workers) % n_workers if N >= n_workers else op_worker[:n_workers]
    W = int(op_worker.max()) + 1
    op_prio = rng.integers(0, max(2, int(N * (1 - p_tie))), size=N).astype(np.int64)
    same = op_worker[src] == op_worker[dst]
    is_flow = (~same & (rng.random(E) > p_nonflow)).astype(np.uint8)
    run_time = np.where(is_flow == 1, np.round(rng.uniform(1e-3, 0.5, size=E), 4), 0.0)
    run_time[(is_flow == 1) & (rng.random(E) < 0.05)] = 0.0           # zero-time flows do occur (2-server sync collectives)
    chan = (op_worker[src].astype(np.int64) * W + op_worker[dst].astype(np.int64))
    keys = np.unique(chan[is_flow == 1])
    cidx = {int(k): i for i, k in enumerate(keys)}
    dep_channel = np.full(E, NO_CHANNEL, dtype=np.uint16)
    for e in np.nonzero(is_flow)[0]:
        if rng.random() > 0.03:                                        # a few flows are left without a channel
            dep_channel[e] = cidx[int(chan[e])]
    dep_prio = rng.integers(0, max(2, int(E * (1 - p_tie))), size=E).astype(np.int64)
    lj = LoweredJob(n_ops=N, n_deps=E, n_workers=W, n_channels=len(keys), num_training_steps=int(rng.integers(1, 60)),
                    model_id=model_id, degree=degree, op_cost=op_cost, op_prio=op_prio, op_worker=op_worker,
                    op_n_parents=n_parents.astype(np.uint16), row_ptr=row_ptr, dep_dst=dst, dep_run_time=run_time,
                    dep_prio=dep_prio, dep_channel=dep_channel, dep_is_flow=is_flow,
                    mount=MountScalars(max_acceptable_jct=float('inf'), part_op_mem=float(N), part_dep_size=float(E),
                                       flow_size=float(is_flow.sum()), n_mounted_workers=W, n_mounted_channels=len(keys)))
    return lj.canonicalise()
