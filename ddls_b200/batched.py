"""Batched gym-like surface over ONE B-episode engine: thousands of ``RampJobPartitioningEnvironment`` rollouts in lock step.

``BatchedRampJobPartitioningEnvironment.reset() -> obs`` / ``.step(actions[B]) -> (obs, reward[B], done[B], info)`` is, per
episode, ``RampJobPartitioningEnvironment.reset / step`` (RJPE:243-274, :300-420): the action is the maximum partition
degree of the queued job (0 = do not place); each op gets ``clamp(even(ceil(cost / quantum)), 1, action)`` sub-ops
(RJPE:332-343); the job is placed by the reference's first-fit rule (ramp_first_fit_place: agents/placers/utils.py:68-582),
partitioned / timed / scheduled / mounted on one-hop channels like the reference's pipeline (ramp_expand_template:
OpPartition, update_dep_run_times, SRPT schedulers, FirstFitDepPlacer), handed to the engine, and the cluster is stepped
until the next job is queued (RJPE:394-395, fused on the device).  Nothing of that is redone per episode:

  * a placement is a pure function of (model, degree, which servers are busy): decisions are cached by that key and the
    B episodes of a step are grouped by it with one ``np.unique`` -- a step of 4,096 episodes calls the native placer a
    handful of times (first-fit blocks repeat), never 4,096 times;
  * a lowered job is a pure function of (model, degree, servers of the block): templates are cached by that key; a miss
    costs one native expansion + one symmetry quotient + one upload (milliseconds), a hit costs nothing;
  * what the policy observes of a job is static per model (node / edge features and the per-graph statistics,
    observation.py:503-567) except a few graph-level numbers: ``obs`` carries the model index of every episode's queued job,
    the dynamic graph features ``[B, 11]`` (the normalised job totals, max-acceptable JCT and fraction, mounted workers and
    running jobs over the cluster size: observation.py:358-498) and the action mask ``[B, |A|]`` (observation.py:80-131).

The per-episode random streams (which model arrives, its max-acceptable-JCT fraction, the inter-arrival gaps) are drawn
up front for ``jobs_per_episode`` arrivals, or supplied (``script=``) -- that is how the tests replay the reference's
recorded episodes in lock step.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import engine as _engine
from .expand import expand_template
from .observation import PARAM_KEYS, _block_shapes_exist, job_arrays
from .synth import ForwardGraph
from .template_builder import RampShape, original_job_totals

SS, EP = _engine.SS, _engine.EP
A100_MEMORY = 80e9                       # devices/processors/gpus/A100.py:17


class _Model:
    """What the environment needs of one job type, computed once."""

    def __init__(self, g: ForwardGraph, quantum: float, num_training_steps: int):
        self.graph = g
        self.n = g.n
        self.mem = [a + p for a, p in zip(g.act, g.par)]
        self.op_mem_total, self.dep_size_total = original_job_totals(g)
        self.n_ops, self.n_deps = 2 * g.n, 2 * len(g.edges) + 1       # the mirrored job's nodes and edges (the join edge n -> n+1)
        self.quantum = quantum
        # summed in the mirrored job's node order (JOB:224-235), as the reference's job details hold it
        self.seq_time = job_arrays(g, num_training_steps)['sequential_completion_time']

    def splits(self, degree: int) -> List[int]:
        return [int(max(1, min(math.ceil(math.ceil(c / self.quantum) / 2) * 2, degree))) for c in self.graph.fwd]   # RJPE:336


def jobs_params(models: Sequence[_Model], frac: Tuple[float, float], num_training_steps: int, max_partitions_per_op_in_observation: int = 1):
    """(min, max) per PARAM_KEYS, by JobsGenerator._init_jobs_params' rules (jobs_generator.py:276-333) over one job of each model:

      * job_total_num_ops: max = int(max * max_partitions_per_op_in_observation)
      * job_total_num_deps: max = int(max / 2 * P * 2) forward + twice that backward (3 * max at P = 1)
      * job_total_dep_sizes: max = max * int(N (N - 1) / 2), N = the largest op count * P (the job made fully connected)
      * every other key: min and max of the values.

    RampJobPartitioningEnvironment never sets max_partitions_per_op_in_observation, so P = 1.  The reference takes the two
    max-acceptable-JCT keys over the max_acceptable_job_completion_time_frac of every job of its sampled pool; that pool is not
    modelled here, so they span the frac distribution's bounds frac = (lo, hi): [lo, hi] and [lo * seq, hi * seq] over the
    models.  Pass the reference's own jobs_params to the environment (``jobs_params=``) to observe exactly what it observes."""
    P = max_partitions_per_op_in_observation
    lo, hi = frac[0], frac[1]
    n_ops, n_deps = [m.n_ops for m in models], [m.n_deps for m in models]
    fwd_deps = int((max(n_deps) / 2) * P * 2)
    max_nodes = max(n_ops) * P
    dep = [m.dep_size_total for m in models]
    seq = [m.seq_time for m in models]
    opm = [m.op_mem_total for m in models]
    macc = [f * s for s in seq for f in (lo, hi)]
    table = {
        'job_total_num_ops': (min(n_ops), int(max(n_ops) * P)),
        'job_total_num_deps': (min(n_deps), fwd_deps + int(fwd_deps * 2)),
        'job_sequential_completion_times': (min(seq), max(seq)),
        'max_acceptable_job_completion_times': (min(macc), max(macc)),
        'max_acceptable_job_completion_time_fracs': (lo, hi),
        'job_total_op_memory_costs': (min(opm), max(opm)),
        'job_total_dep_sizes': (min(dep), max(dep) * int(max_nodes * (max_nodes - 1) / 2)),
        'job_num_training_steps': (num_training_steps, num_training_steps),
    }
    return [(float(table[k][0]), float(table[k][1])) for k in PARAM_KEYS]


_default_jobs_params = jobs_params              # the environment's constructor argument of the same name shadows it

PLACE_SMEM_PER_WARP = 12288                     # include/ramp_b200.h RAMP_ENV_PLACE_SMEM_PER_WARP


def candidate_blocks(shape: Tuple[int, int, int], max_degree: int):
    """The blocks RampFirstFitOpPlacer tries for an op of d sub-ops, d = 1 and every even d <= max_degree, in its (block shape,
    origin) order (utils.py:333-383, 394-443, 491-530), each as its servers' indices ((c * R + r) * S + s) in get_block order.
    Blocks check_block always rejects (a server outside the cluster) are left out.  Returns (cand_ptr, blocks): the blocks of
    degree d are blocks[cand_ptr[d]:cand_ptr[d + 1]]."""
    from .placer import _block_shapes, _factor_pairs, _get_block
    index = {(c, r, s): (c * shape[1] + r) * shape[2] + s for c in range(shape[0]) for r in range(shape[1]) for s in range(shape[2])}
    cand_ptr, blocks = [0, 0], []
    for d in range(1, max_degree + 1):
        if d == 1 or d % 2 == 0:
            for bs in _block_shapes(_factor_pairs(d), shape) + [(d, d, -1), (d, 1, 1)]:
                I, J_, K = (shape[0] - bs[0]) + 1, (shape[1] - bs[1]) + 1, (shape[2] - bs[2]) + 1
                if I <= 0 or J_ <= 0 or K <= 0:
                    continue
                for i in range(I):
                    for j in range(J_):
                        for k in range(K):
                            block = _get_block(bs[0], bs[1], bs[2], shape, (i, j, k))
                            if any(sv not in index for sv in block) or len(set(block)) != d:
                                continue                                                             # check_block fails on it
                            blocks.append([index[sv] for sv in block])
        cand_ptr.append(len(blocks))
    return cand_ptr, blocks


def canonical_mask(coords, shape: Tuple[int, int, int], n_words: int):
    """The servers `coords` with each coordinate axis relabelled 0, 1, ... over the values it takes (the order-preserving
    relabelling of the template key of ``_place_many``), as a bit set over the servers of `shape`: what ramp_env_place_kernel
    looks the lowered job up by.  Two server sets have the same mask exactly when they have the same template key."""
    ranks = [{v: i for i, v in enumerate(sorted({c[ax] for c in coords}))} for ax in range(3)]
    words = [0] * n_words
    for c in coords:
        j = (ranks[0][c[0]] * shape[1] + ranks[1][c[1]]) * shape[2] + ranks[2][c[2]]
        words[j >> 6] |= 1 << (j & 63)
    return tuple(words)


def placer_tables(models: Sequence['_Model'], max_degree: int):
    """What ramp_env_place_kernel needs of every model (include/ramp_b200.h ramp_env_placer_tables_t): per model its ops in
    topo_sort order (utils.py:100-115, as ramp_first_fit_place orders them), the parents of each op in the graph's edge order, the
    bytes of each op, and the sub-ops of each op at every degree.  Op indices are within the model, from 0."""
    op_ptr, topo, par_ptr, parents, need = [0], [], [0], [], []
    for model in models:
        g, n = model.graph, model.n
        par = [[] for _ in range(n + 1)]
        children = [[] for _ in range(n + 1)]
        for (u, v) in g.edges:
            par[v].append(u)
            children[u].append(v)
        left = [list(p) for p in par]
        seq = [v for v in range(1, n + 1) if not left[v]]
        for v in seq:                                         # seq grows while it is walked: the queue of topo_sort
            for c in children[v]:
                left[c].remove(v)
                if not left[c]:
                    seq.append(c)
        if len(seq) != n:
            raise ValueError(f'model {g.name}: the graph has a cycle')
        topo += [v - 1 for v in seq]
        for v in range(1, n + 1):
            parents += [u - 1 for u in par[v]]
            par_ptr.append(len(parents))
        need += model.mem
        op_ptr.append(op_ptr[-1] + n)
    splits = np.ones((max_degree + 1, op_ptr[-1]), dtype=np.int32)
    for d in range(1, max_degree + 1):
        splits[d] = np.concatenate([np.asarray(m.splits(d), dtype=np.int32) for m in models])
    return dict(op_ptr=np.asarray(op_ptr, dtype=np.int32), topo=np.asarray(topo, dtype=np.int32),
                par_ptr=np.asarray(par_ptr, dtype=np.int32), parents=np.asarray(parents, dtype=np.int32).reshape(-1),
                need=np.asarray(need, dtype=np.float64), splits=splits)


def place_smem_per_warp(n_workers: int, max_ops: int) -> int:
    """Shared memory ramp_env_place_kernel keeps per warp: free memory of every server (and 8 doubles of slack for the template
    key), one candidate index per op of the largest model."""
    return (8 * (n_workers + 8) + 4 * max_ops + 7) // 8 * 8


class BatchedRampJobPartitioningEnvironment:
    def __init__(self, shape: Tuple[int, int, int], graphs: Sequence[ForwardGraph], n_episodes: int, jobs_per_episode: int = 8,
                 max_partitions_per_op: int = 16, min_op_run_time_quantum: float = 0.01, num_training_steps: int = 50,
                 interarrival=('fixed', 1000.0), frac=(0.1, 1.0, 2), max_simulation_run_time: float = float('inf'),
                 fail_reward: float = -1, success_reward: float = 1, device: int = 0, seed: int = 0,
                 run_times: str = 'reference', apply_action_mask: bool = True, script: Optional[dict] = None,
                 memo_mode: int = _engine.MEMO_REFERENCE, jobs_params: Optional[dict] = None, machine_epsilon: float = 1e-7):
        """jobs_params: the normalisers of the observation's job features, as the reference's ``JobsGenerator.jobs_params`` holds
        them (``min_<key>`` / ``max_<key>`` for the keys of observation.PARAM_KEYS); the keys it gives replace the defaults of
        ``jobs_params(models, ...)``.  machine_epsilon: added to a normalised feature that comes out negative (observation.py:441-444,
        493-496), as RampJobPartitioningObservation does."""
        self.shape = RampShape(*shape)
        self.W = self.shape.n_workers
        self.B, self.J = int(n_episodes), int(jobs_per_episode)
        self.max_partitions_per_op = int(max_partitions_per_op)
        self.num_training_steps = num_training_steps
        self.models = [_Model(g, min_op_run_time_quantum, num_training_steps) for g in graphs]
        self.interarrival, self.frac_dist = interarrival, frac
        self.max_simulation_run_time = float(max_simulation_run_time)
        self.fail_reward, self.success_reward = fail_reward, success_reward
        self.apply_action_mask = apply_action_mask
        self.run_times = run_times
        self.rng = np.random.default_rng(seed)
        self.script = script
        self.eng = _engine.RampEngine(n_episodes=self.B, n_cluster_workers=self.W, max_jobs=self.J, device=device,
                                      memo_mode=memo_mode, trace_cap=8192, max_simulation_run_time=self.max_simulation_run_time,
                                      env_step_stats=True)
        self.n_words = (self.W + 63) // 64
        self._servers = [(c, r, s) for c in range(self.shape.c) for r in range(self.shape.r) for s in range(self.shape.s)]
        self._server_index = {sv: i for i, sv in enumerate(self._servers)}
        # action set (observation.py:80-131): 0..max_partitions_per_op; which actions have a RAMP-symmetric block shape at all
        self.action_set = np.arange(self.max_partitions_per_op + 1, dtype=np.int16)
        self._shape_ok = np.array([True] + [(a == 1) or (a % 2 == 0 and _block_shapes_exist(a, shape))
                                            for a in range(1, self.max_partitions_per_op + 1)])
        # caches
        self._placement_cache: Dict[tuple, tuple] = {}       # (model, degree, busy words...) -> (template id | -1, mask words)
        self._template_cache: Dict[tuple, int] = {}          # (model, degree, block geometry) -> template id
        self._t_mount: List[tuple] = []                      # per template id: (seq_time, part_op_mem, part_dep, flow, n_workers, n_channels)
        self._t_arrays = None
        self.stats = {'placer_calls': 0, 'expansions': 0, 'placement_hits': 0}
        self.machine_epsilon = float(machine_epsilon)
        self._jobs_params = _default_jobs_params(self.models, frac, num_training_steps)
        for i, k in enumerate(PARAM_KEYS):
            if jobs_params is not None and f'min_{k}' in jobs_params and f'max_{k}' in jobs_params:
                self._jobs_params[i] = (float(jobs_params[f'min_{k}']), float(jobs_params[f'max_{k}']))

    # ---- arrival streams ------------------------------------------------------------------------------------------
    def _draw_streams(self):
        B, J, M = self.B, self.J, len(self.models)
        if self.script is not None:
            self.model_of = np.asarray(self.script['model'], dtype=np.int64).reshape(B, J)
            gaps = np.asarray(self.script['gap'], dtype=np.float64).reshape(B, J)
            self.frac = np.asarray(self.script.get('frac', np.ones((B, J))), dtype=np.float64).reshape(B, J)
            self.macc_override = (np.asarray(self.script['max_acceptable_jct'], dtype=np.float64).reshape(B, J)
                                  if 'max_acceptable_jct' in self.script else None)
        else:
            self.model_of = self.rng.integers(0, M, size=(B, J))
            kind = self.interarrival[0]
            if kind == 'fixed':
                gaps = np.full((B, J), float(self.interarrival[1]))
            elif kind == 'exponential':
                gaps = self.rng.exponential(float(self.interarrival[1]), size=(B, J))
            else:
                raise Exception(f'unknown inter-arrival distribution {kind}')
            gaps[:, J - 1] = np.inf                              # no job after the last one (jobs_generator.py:270-272)
            lo, hi, dec = self.frac_dist
            self.frac = np.round(self.rng.uniform(lo, hi, size=(B, J)), dec)
            self.macc_override = None
        arr = np.zeros((B, J), dtype=_engine.ARRIVAL_DTYPE)
        arr['interarrival'] = gaps
        arr['orig_op_mem'] = np.array([m.op_mem_total for m in self.models])[self.model_of]
        arr['orig_dep_size'] = np.array([m.dep_size_total for m in self.models])[self.model_of]
        return arr

    # ---- RJPE.reset ----------------------------------------------------------------------------------------------
    def reset(self):
        self.arrivals = self._draw_streams()
        self.eng.reset(self.arrivals)
        B, J = self.B, self.J
        self.busy = np.zeros((B, self.n_words), dtype=np.uint64)
        self.job_mask = np.zeros((B, J, self.n_words), dtype=np.uint64)
        self.status = np.zeros((B, J), dtype=np.int32)
        self.status[:, 0] = _engine.JS_QUEUED
        self.queued = np.zeros(B, dtype=np.int64)                 # RCE:280-281: job 0 is queued
        self.done = np.zeros(B, dtype=bool)
        self.n_running = np.zeros(B, dtype=np.int64)
        self.job_template = np.full((B, J), -1, dtype=np.int32)    # template each accepted job was mounted with
        self.episode_return = np.zeros(B, dtype=np.float64)        # sum of the rewards since the reset
        self.step_counter = 0
        return self._observe()

    # ---- placement + lowering, cached ------------------------------------------------------------------------------
    def _free_count(self):
        return self.W - np.bitwise_count(self.busy).sum(axis=1).astype(np.int64)

    def action_mask(self):
        """[B, |A|] validity of every action for the queued job (observation.py:80-131)."""
        free = self._free_count()
        a = self.action_set.astype(np.int64)[None, :]
        ok = (a <= free[:, None]) & self._shape_ok[None, :]
        ok[:, 0] = True
        return ok

    def _c_graph(self, m: int):
        """ramp_forward_graph_t of model m (built once; only the memory costs and the edges matter to the placer)."""
        import ctypes as C
        from .expand import _FwdGraph
        model = self.models[m]
        if not hasattr(model, '_cg'):
            mem = np.ascontiguousarray(model.mem, dtype=np.float64)
            zero = np.zeros(model.n, dtype=np.float64)
            es = np.ascontiguousarray([u for (u, _) in model.graph.edges], dtype=np.int32)
            ed = np.ascontiguousarray([v for (_, v) in model.graph.edges], dtype=np.int32)
            model._cg_keep = (mem, zero, es, ed)
            model._cg = _FwdGraph(model.n, len(model.graph.edges), zero.ctypes.data, zero.ctypes.data, mem.ctypes.data, zero.ctypes.data,
                                  es.ctypes.data, ed.ctypes.data)
        return model._cg

    def _place_many(self, m: int, degree: int, busy_rows: np.ndarray):
        """First-fit placement of model m at `degree` on every cluster state of busy_rows [n, n_words] (one native call), then the
        template of each resulting block (cached).  Fills the placement cache."""
        import ctypes as C
        L = _engine.load_library()
        L.ramp_first_fit_place_many.restype = C.c_int
        L.ramp_first_fit_place_many.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]
        model = self.models[m]
        n = len(busy_rows)
        busy_rows = np.ascontiguousarray(busy_rows, dtype=np.uint64)
        splits = np.ascontiguousarray(model.splits(degree), dtype=np.int32)
        shape = (C.c_int32 * 3)(self.shape.c, self.shape.r, self.shape.s)
        masks = np.zeros((n, self.n_words), dtype=np.uint64)
        ok = np.zeros(n, dtype=np.uint8)
        g = self._c_graph(m)
        _engine._check(L.ramp_first_fit_place_many(C.byref(g), splits.ctypes.data, shape, A100_MEMORY, n, self.n_words,
                                                  busy_rows.ctypes.data, masks.ctypes.data, ok.ctypes.data))
        self.stats['placer_calls'] += n
        for k in range(n):
            key = (m, degree) + tuple(int(x) for x in busy_rows[k])
            if not ok[k]:                                          # the reference leaves the job out of the Action: blocked (RCE:914-919)
                self._placement_cache[key] = (-1, (0,) * self.n_words)
                continue
            words = tuple(int(x) for x in masks[k])
            coords = [self._servers[i] for i in range(self.W) if (words[i >> 6] >> (i & 63)) & 1]
            # the lowered job depends on the block only through which servers share a communication group / rack / server index
            # (collective times, actions/utils.py:168-245; one-to-one transfers only test equality): blocks that are equal after an
            # order-preserving relabelling of each coordinate axis give byte-identical jobs (tests/test_expand_native.py)
            ranks = [{v: i for i, v in enumerate(sorted({c[ax] for c in coords}))} for ax in range(3)]
            tkey = (m, degree, tuple((ranks[0][c[0]], ranks[1][c[1]], ranks[2][c[2]]) for c in coords))
            tid = self._template_cache.get(tkey)
            if tid is None:
                self.stats['expansions'] += 1
                lj = expand_template(model.graph, degree, self.shape, quantum=model.quantum,
                                     num_training_steps=self.num_training_steps, model_id=m, run_times=self.run_times, coords=coords)
                tid = self.eng.register_template(lj)
                self._template_cache[tkey] = tid
                mt = lj.mount
                while len(self._t_mount) <= tid:
                    self._t_mount.append(None)
                self._t_mount[tid] = (lj.seq_time, mt.part_op_mem, mt.part_dep_size, mt.flow_size, mt.n_mounted_workers, mt.n_mounted_channels)
                self._t_arrays = None
            self._placement_cache[key] = (tid, words)

    def _mount_arrays(self):
        if self._t_arrays is None:
            rows = [r if r is not None else (0.0,) * 6 for r in self._t_mount]
            self._t_arrays = np.array(rows, dtype=np.float64).reshape(-1, 6) if rows else np.zeros((0, 6))
        return self._t_arrays

    # ---- RJPE.step -----------------------------------------------------------------------------------------------
    def step(self, actions):
        B, J = self.B, self.J
        actions = np.asarray(actions, dtype=np.int64).reshape(B)
        live = ~self.done
        q = self.queued
        if np.any(live & (q < 0)):
            raise Exception('an episode that is not done has no queued job (RJPE:394-395 keeps stepping until there is one)')
        mask = self.action_mask()
        bad_set = live & ((actions < 0) | (actions > self.max_partitions_per_op))
        if np.any(bad_set):
            b = int(np.nonzero(bad_set)[0][0])
            raise Exception(f'Action {int(actions[b])} not in action set {self.action_set.tolist()}.')                 # RJPE:314-316
        invalid = live & ~mask[np.arange(B), np.clip(actions, 0, self.max_partitions_per_op)]
        if np.any(invalid):
            if self.apply_action_mask:
                b = int(np.nonzero(invalid)[0][0])
                raise Exception(f'Action {int(actions[b])} is invalid given action mask {mask[b].astype(int).tolist()}.')  # RJPE:317-319
            actions = np.where(invalid, 0, actions)                                                                        # RJPE:320-322
        qq = np.clip(q, 0, J - 1)
        m_of = self.model_of[np.arange(B), qq]
        # ---- group the episodes by (model, degree, busy servers): one placement decision per group ----
        tid = np.full(B, -1, dtype=np.int32)
        mask_words = np.zeros((B, self.n_words), dtype=np.uint64)
        sel = np.nonzero(live & (actions > 0))[0]
        if len(sel):
            keys = np.concatenate([m_of[sel, None].astype(np.uint64), actions[sel, None].astype(np.uint64), self.busy[sel]], axis=1)
            uniq, inv = np.unique(keys, axis=0, return_inverse=True)
            inv = inv.reshape(-1)
            u_tid = np.empty(len(uniq), dtype=np.int32)
            u_words = np.zeros((len(uniq), self.n_words), dtype=np.uint64)
            rows = [tuple(int(x) for x in row) for row in uniq]
            miss = [k for k, row in enumerate(rows) if row not in self._placement_cache]
            self.stats['placement_hits'] += len(rows) - len(miss)
            by_md = {}
            for k in miss:
                by_md.setdefault(rows[k][:2], []).append(k)
            for (m_, d_), ks in by_md.items():
                self._place_many(m_, d_, uniq[ks][:, 2:])
            for k, row in enumerate(rows):
                t, words = self._placement_cache[row]
                u_tid[k] = t
                u_words[k] = np.array(words, dtype=np.uint64)
            tid[sel] = u_tid[inv]
            mask_words[sel] = u_words[inv]
        # ---- action rows ----
        act = self.eng.make_actions()
        act['flags'] = np.where(live, 0, _engine.ACT_SKIP)
        placed = tid >= 0
        if placed.any():
            mt = self._mount_arrays()[tid[placed]]
            fr = self.frac[np.arange(B), qq][placed]
            macc = fr * mt[:, 0]
            if self.macc_override is not None:
                ov = self.macc_override[np.arange(B), qq][placed]
                macc = np.where(np.isnan(ov), macc, ov)
            act['max_acceptable_jct'][placed] = macc
            act['part_op_mem'][placed] = mt[:, 1]
            act['part_dep_size'][placed] = mt[:, 2]
            act['flow_size'][placed] = mt[:, 3]
            act['n_mounted_workers'][placed] = mt[:, 4].astype(np.int32)
            act['n_mounted_channels'][placed] = mt[:, 5].astype(np.int32)
        act['template_id'] = tid
        stats, ncs = self.eng.step(act, fuse_empty_steps=True, want_cluster_steps=True)
        self.eng.check_status()
        rec = self.eng.job_records()
        ep = self.eng.episode_state()
        status = rec['status']
        # ---- reward (rewards/job_acceptance.py): the job counts as placed unless it was blocked by the end of the FIRST cluster
        #      step (RJPE:379-391); a lookahead-blocked job has no lookahead results in its record ----
        rq = rec[np.arange(B), qq]
        accepted = placed & (rq['jct'] != 0.0)
        blocked_in_action_step = accepted & (rq['status'] == _engine.JS_BLOCKED) & (ncs == 1)
        reward = np.where(accepted & ~blocked_in_action_step, self.success_reward, self.fail_reward).astype(np.float64)
        reward[~live] = 0.0
        # ---- occupancy: servers of the jobs that are running now ----
        acc = np.nonzero(accepted)[0]
        self.job_mask[acc, qq[acc]] = mask_words[acc]
        self.job_template[acc, qq[acc]] = tid[acc]
        self.episode_return += reward
        running = (status == _engine.JS_RUNNING)
        self.busy = np.bitwise_or.reduce(np.where(running[:, :, None], self.job_mask, np.uint64(0)), axis=1)
        self.n_running = running.sum(axis=1)
        self.status = status
        self.queued = ep[:, EP['queued_job']].astype(np.int64)
        self.done = ep[:, EP['done']] != 0
        self.last_stats, self.last_cluster_steps = stats, ncs
        self.step_counter += 1
        info = {'template_id': tid, 'cluster_steps': ncs, 'accepted': accepted}
        return self._observe(), reward, self.done.copy(), info

    # ---- EvalLoop's episode statistics ----------------------------------------------------------------------------
    def _episode_tables(self):
        return self.job_template, self.episode_return

    def episode_stats(self):
        """RampClusterEnvironment.episode_stats of every episode, keyed by the reference's names (RCE:1086-1167, 1466-1540), plus
        EvalLoop's ``return`` (loops/eval_loop.py:26-134).  Every scalar is an array [B] (``engine.ES_FIELDS``: the finalised
        episode means over every cluster step, fused ones included; episodes that are not done hold the same formulas over the
        episode so far).  The per-job lists are lists of B arrays in completion order (event order): ``job_completion_time``,
        ``job_completion_time_speedup``, ``job_communication_overhead_time``, ``job_computation_overhead_time``,
        ``jobs_completed_mean_mounted_worker_utilisation_frac``, ``jobs_completed_num_mounted_workers`` / ``_channels``,
        ``jobs_completed_max_acceptable_job_completion_time``, ``jobs_blocked_max_acceptable_job_completion_time``, with the job
        indices in ``completed_job_idxs`` / ``blocked_job_idxs``.  Reads the [B][J] tables back once: call it when episodes end."""
        ES = _engine.ES
        rows = self.eng.episode_stats()
        job_template, ret = self._episode_tables()
        rec = self.eng.job_records()
        out = {}
        for k in _engine.ES_FIELDS:
            col = rows[:, ES[k]]
            out[k] = col.astype(np.int64) if k in _engine.ES_COUNTS else col.astype(bool) if k == 'done' else col.copy()
        out['return'] = np.array(ret, dtype=np.float64)
        mounts = self._mount_arrays()
        if not len(mounts):
            mounts = np.zeros((1, 6))
        seq = np.array([m.seq_time for m in self.models], dtype=np.float64)
        # every [B][J] table in each episode's event order
        order = np.argsort(rec['event_seq'], axis=1, kind='stable')
        r = np.take_along_axis(rec, order, axis=1)
        tid = np.take_along_axis(job_template, order, axis=1)
        model_of = np.take_along_axis(self.model_of, order, axis=1)
        # the job's max acceptable JCT as the action row carried it: the override, else frac x the sequential time of the template
        # it was mounted with (of its model when it was never mounted)
        macc = np.take_along_axis(self.frac, order, axis=1) * np.where(tid >= 0, mounts[np.maximum(tid, 0), 0], seq[model_of])
        if self.macc_override is not None:
            ov = np.take_along_axis(self.macc_override, order, axis=1)
            macc = np.where(np.isnan(ov), macc, ov)
        comp, blk = r['status'] == _engine.JS_COMPLETED, r['status'] == _engine.JS_BLOCKED

        def per_episode(mask, values):
            return np.split(values[mask], np.cumsum(mask.sum(axis=1))[:-1])
        jct = r['time_completed'] - r['time_arrived']
        mt = mounts[np.maximum(tid, 0)]
        with np.errstate(divide='ignore', invalid='ignore'):
            speedup = seq[model_of] / jct
        lists = {'job_completion_time': per_episode(comp, jct), 'job_completion_time_speedup': per_episode(comp, speedup),
                 'job_communication_overhead_time': per_episode(comp, r['comm']),
                 'job_computation_overhead_time': per_episode(comp, r['comp']),
                 'jobs_completed_mean_mounted_worker_utilisation_frac': per_episode(comp, r['util']),
                 'jobs_completed_num_mounted_workers': per_episode(comp, mt[..., 4].astype(np.int64)),
                 'jobs_completed_num_mounted_channels': per_episode(comp, mt[..., 5].astype(np.int64)),
                 'jobs_completed_max_acceptable_job_completion_time': per_episode(comp, macc),
                 'jobs_blocked_max_acceptable_job_completion_time': per_episode(blk, macc),
                 'completed_job_idxs': per_episode(comp, order.astype(np.int64)), 'blocked_job_idxs': per_episode(blk, order.astype(np.int64))}
        out.update(lists)
        return out

    def env_step_stats(self):
        """EvalLoop's results['step_stats'] entries for every episode's last env-step (loops/eval_loop.py:50-100), as [B] arrays keyed
        by the cluster's steps_log names in its order (``engine.ENV_STEP_STATS``): every key reduced by the step kernel over the
        cluster steps of the env-step, the fused empty ones included -- step_start_time the first value, step_end_time and
        step_counter the last, 'mean' keys the mean, the others the sum; the per-tick utilisation lists the mean over every entry.
        A finished episode keeps its last env-step's row.  ``step()``'s return value does not carry it."""
        return _engine.env_step_columns(self.eng.env_step_stats())

    # ---- observations ---------------------------------------------------------------------------------------------
    def jobs_params(self):
        """(min, max) per PARAM_KEYS: the normalisers of the observation's job features (``jobs_params(models, ...)`` or the
        reference's table given to the constructor)."""
        return self._jobs_params

    def _observe(self):
        B = self.B
        qq = np.clip(self.queued, 0, self.J - 1)
        m_of = self.model_of[np.arange(B), qq]
        fr = self.frac[np.arange(B), qq]
        P = self._jobs_params

        def norm(x, k):
            lo, hi = P[PARAM_KEYS.index(k)]
            return (x - lo) / (hi - lo) if hi - lo != 0 else np.ones_like(x, dtype=np.float64)
        seq = np.array([m.seq_time for m in self.models])[m_of]
        n_ops = np.array([float(m.n_ops) for m in self.models])[m_of]
        n_deps = np.array([float(m.n_deps) for m in self.models])[m_of]
        opm = np.array([m.op_mem_total for m in self.models])[m_of]
        dps = np.array([m.dep_size_total for m in self.models])[m_of]
        mounted = self.W - self._free_count()
        dyn = np.stack([norm(n_ops, 'job_total_num_ops'), norm(n_deps, 'job_total_num_deps'),
                        norm(seq, 'job_sequential_completion_times'), norm(fr * seq, 'max_acceptable_job_completion_times'),
                        norm(fr, 'max_acceptable_job_completion_time_fracs'), fr, norm(opm, 'job_total_op_memory_costs'),
                        norm(dps, 'job_total_dep_sizes'),
                        norm(np.full(B, float(self.num_training_steps)), 'job_num_training_steps'),
                        mounted / self.W, self.n_running / self.W], axis=1)
        dyn = np.where(dyn < 0, dyn + self.machine_epsilon, dyn).astype(np.float32)     # observation.py:441-444, 493-496
        mask = self.action_mask()
        return {'model': m_of.astype(np.int32), 'graph_features_dynamic': dyn, 'action_set': self.action_set,
                'action_mask': mask.astype(np.int16), 'queued_job': self.queued.copy(), 'done': self.done.copy()}

    def close(self):
        self.eng.close()


class DeviceRampJobPartitioningEnvironment(BatchedRampJobPartitioningEnvironment):
    """The same environment with the per-step decision and bookkeeping ON THE DEVICE (include/ramp_b200.h: ramp_env_*): first-fit
    placement over host-enumerated candidate blocks (SURVEY 8f-4), template lookup by (model, degree, block geometry), action
    rows, reward, occupancy, dynamic observation features and action mask (8f-2) are kernels with one thread per episode; a step
    is ``ramp_env_decide`` -> ``ramp_env_advance`` and, through ``step``, one read-back of the outputs.  ``device_buffers()`` gives
    the raw device pointers for a policy that lives on the GPU (then nothing crosses PCIe).  The host is asked only for what the
    tables cannot decide: jobs whose ops take different numbers of sub-ops, and the first use of a block geometry (it lowers the
    job natively, registers it and fills the table).

    place_on_device=True places the jobs whose ops split unevenly on the device too (ramp_env_place_kernel: the same first-fit
    placer, one warp per episode) and finds their lowered job by the canonical mask of the servers used; the host then only
    lowers each new (model, degree, canonical mask) once, and a warmed environment never calls the host's placer.  It needs
    ``place_smem_per_warp(servers, ops of the largest model)`` <= PLACE_SMEM_PER_WARP bytes; past that the environment warns and
    keeps the host path (``self.place_on_device`` is then False)."""

    def __init__(self, *args, prewarm: bool = False, place_on_device: bool = False, **kw):
        import ctypes as C
        super().__init__(*args, **kw)
        D, nw, shape = self.max_partitions_per_op, self.n_words, (self.shape.c, self.shape.r, self.shape.s)
        self._geom_index: Dict[tuple, int] = {}
        self._geom_example: Dict[tuple, list] = {}          # (degree, geometry index) -> one block with that geometry
        cand_ptr, self._cand_blocks = candidate_blocks(shape, D)
        cand_mask, cand_geom = [], []
        for blk in self._cand_blocks:
            words = [0] * nw
            for ix in blk:
                words[ix >> 6] |= (1 << (ix & 63))
            cand_mask.append(words)
            coords = [self._servers[ix] for ix in sorted(blk)]
            gi = self._geometry(coords)
            cand_geom.append(gi)
            self._geom_example.setdefault((len(blk), gi), coords)
        self._n_geoms = max(len(self._geom_index), 1)
        M = len(self.models)
        uniform = np.zeros((M, D + 1), dtype=np.uint8)
        for m, model in enumerate(self.models):
            sources = set(range(1, model.n + 1)) - {v for (_, v) in model.graph.edges}
            for d in range(1, D + 1):
                if (d == 1 or d % 2 == 0) and all(s == d for s in model.splits(d)) and len(sources) == 1 \
                        and sum(model.mem) <= d * A100_MEMORY:
                    uniform[m, d] = 1
        self._uniform = uniform
        P = self._jobs_params
        mp = np.array([[mo.seq_time, mo.n_ops, mo.n_deps, mo.op_mem_total, mo.dep_size_total] for mo in self.models], dtype=np.float64)
        keep = dict(cand_ptr=np.ascontiguousarray(cand_ptr, dtype=np.int32),
                    cand_mask=np.ascontiguousarray(cand_mask, dtype=np.uint64).reshape(-1, nw),
                    cand_geom=np.ascontiguousarray(cand_geom, dtype=np.int32), uniform=np.ascontiguousarray(uniform),
                    shape_ok=np.ascontiguousarray(self._shape_ok, dtype=np.uint8), mp=np.ascontiguousarray(mp),
                    jp=np.ascontiguousarray(P, dtype=np.float64).reshape(8, 2))

        class _Cfg(C.Structure):
            _fields_ = [('shape', C.c_int32 * 3), ('n_models', C.c_int32), ('max_degree', C.c_int32), ('n_geoms', C.c_int32),
                        ('jobs_per_episode', C.c_int32), ('n_words', C.c_int32), ('apply_action_mask', C.c_int32),
                        ('num_training_steps', C.c_int32), ('fail_reward', C.c_double), ('success_reward', C.c_double),
                        ('machine_epsilon', C.c_double),
                        ('cand_ptr', C.c_void_p), ('cand_mask', C.c_void_p), ('cand_geom', C.c_void_p), ('uniform', C.c_void_p),
                        ('shape_ok', C.c_void_p), ('model_params', C.c_void_p), ('jobs_params', C.c_void_p)]
        cfg = _Cfg((C.c_int32 * 3)(*shape), M, D, self._n_geoms, self.J, nw, 1 if self.apply_action_mask else 0, self.num_training_steps,
                   float(self.fail_reward), float(self.success_reward), self.machine_epsilon,
                   keep['cand_ptr'].ctypes.data, keep['cand_mask'].ctypes.data,
                   keep['cand_geom'].ctypes.data, keep['uniform'].ctypes.data, keep['shape_ok'].ctypes.data, keep['mp'].ctypes.data,
                   keep['jp'].ctypes.data)
        L = self.eng._L
        for name in ('ramp_env_create', 'ramp_env_set_template', 'ramp_env_reset', 'ramp_env_buffers', 'ramp_env_decide', 'ramp_env_patch',
                     'ramp_env_advance', 'ramp_env_read'):
            getattr(L, name).restype = C.c_int
        L.ramp_env_create.argtypes = [C.c_void_p, C.c_void_p]
        L.ramp_env_set_template.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
        L.ramp_env_reset.argtypes = [C.c_void_p] * 5
        L.ramp_env_buffers.argtypes = [C.c_void_p, C.c_void_p]
        L.ramp_env_decide.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ramp_env_patch.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]
        L.ramp_env_advance.argtypes = [C.c_void_p]
        L.ramp_env_read.argtypes = [C.c_void_p] * 6
        _engine._check(L.ramp_env_create(self.eng._h, C.byref(cfg)))
        self._table_set = set()
        B, A = self.B, D + 1
        # page-locked host arrays for the per-step transfers (actions in; reward / done / observation out): numpy views
        mirror = self._buffers('ramp_env_host_mirror')

        def view(ptr, ctype, shape):
            n = int(np.prod(shape))
            return np.ctypeslib.as_array((ctype * n).from_address(ptr)).reshape(shape)
        self._actions_pinned = view(mirror['actions'], C.c_int32, (B,))
        self._reward = view(mirror['reward'], C.c_double, (B,))
        self._done = view(mirror['done'], C.c_uint8, (B,))
        self._qmodel = view(mirror['queued_model'], C.c_int32, (B,))
        self._obs_dyn = view(mirror['obs_dynamic'], C.c_float, (B, 11))
        self._mask = view(mirror['action_mask'], C.c_uint8, (B, A))
        self._need = np.zeros(B, dtype=np.int32)
        self._prewarmed = False
        self._decides_all = None
        self.place_on_device = bool(place_on_device)
        self._geom_mask_set = set()                         # (model, degree, canonical mask) entries given to the device table
        if self.place_on_device:
            self._set_placer_tables(cand_ptr)
        if prewarm:
            self.prewarm()

    def _set_placer_tables(self, cand_ptr):
        import ctypes as C
        import warnings
        need = place_smem_per_warp(self.W, max(m.n for m in self.models))
        if need > PLACE_SMEM_PER_WARP:
            warnings.warn(f'place_on_device: {self.W} servers and {max(m.n for m in self.models)} ops need {need} bytes of shared '
                          f'memory per warp, more than {PLACE_SMEM_PER_WARP}; jobs whose ops split unevenly stay with the host placer')
            self.place_on_device = False
            return
        t = placer_tables(self.models, self.max_partitions_per_op)
        t['cand_offset'] = np.ascontiguousarray(np.cumsum([0] + [len(b) for b in self._cand_blocks]), dtype=np.int32)
        t['cand_servers'] = np.ascontiguousarray([ix for b in self._cand_blocks for ix in b], dtype=np.int32).reshape(-1)
        assert int(t['cand_offset'].shape[0]) == cand_ptr[-1] + 1

        class _Tables(C.Structure):
            _fields_ = [('n_ops_total', C.c_int32), ('memory_capacity', C.c_double)] + [
                (k, C.c_void_p) for k in ('op_ptr', 'topo', 'par_ptr', 'parents', 'need', 'splits', 'cand_offset', 'cand_servers')]
        self._placer_keep = {k: np.ascontiguousarray(v) for k, v in t.items()}
        tab = _Tables(int(t['op_ptr'][-1]), A100_MEMORY, *[self._placer_keep[k].ctypes.data for k in
                      ('op_ptr', 'topo', 'par_ptr', 'parents', 'need', 'splits', 'cand_offset', 'cand_servers')])
        L = self.eng._L
        L.ramp_env_set_placer_tables.restype = C.c_int
        L.ramp_env_set_placer_tables.argtypes = [C.c_void_p, C.c_void_p]
        L.ramp_env_set_geometry_template.restype = C.c_int
        L.ramp_env_set_geometry_template.argtypes = [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
        _engine._check(L.ramp_env_set_placer_tables(self.eng._h, C.byref(tab)))

    def _canonical_mask(self, coords):
        return canonical_mask(coords, (self.shape.c, self.shape.r, self.shape.s), self.n_words)

    def prewarm(self):
        """Lowers and registers the job of every (model, degree, block geometry) the device can choose, so that no step waits
        for a native expansion (each costs 1-60 ms once)."""
        import ctypes as C
        for (d, gi), block in sorted(self._geom_example.items()):
            for m, model in enumerate(self.models):
                if not self._uniform[m, d] or (m, d, gi) in self._table_set:
                    continue
                ranks = [{v: i for i, v in enumerate(sorted({c[ax] for c in block}))} for ax in range(3)]
                tkey = (m, d, tuple((ranks[0][c[0]], ranks[1][c[1]], ranks[2][c[2]]) for c in block))
                tid = self._template_cache.get(tkey)
                if tid is None:
                    self.stats['expansions'] += 1
                    lj = expand_template(model.graph, d, self.shape, quantum=model.quantum, num_training_steps=self.num_training_steps,
                                         model_id=m, run_times=self.run_times, coords=block)
                    tid = self.eng.register_template(lj)
                    self._template_cache[tkey] = tid
                    mt = lj.mount
                    while len(self._t_mount) <= tid:
                        self._t_mount.append(None)
                    self._t_mount[tid] = (lj.seq_time, mt.part_op_mem, mt.part_dep_size, mt.flow_size, mt.n_mounted_workers, mt.n_mounted_channels)
                    self._t_arrays = None
                mt = np.array(self._t_mount[tid], dtype=np.float64)
                _engine._check(self.eng._L.ramp_env_set_template(self.eng._h, m, d, gi, tid, mt.ctypes.data))
                self._table_set.add((m, d, gi))
        self._prewarmed = True

    @property
    def _device_decides_everything(self):
        if not self._prewarmed:
            return False
        if self._decides_all is None:
            valid = [d for d in range(1, self.max_partitions_per_op + 1) if self._shape_ok[d] and d <= self.W]
            self._decides_all = all(bool(self._uniform[m, d]) for m in range(len(self.models)) for d in valid)
        return self._decides_all

    def _geometry(self, coords):
        ranks = [{v: i for i, v in enumerate(sorted({c[ax] for c in coords}))} for ax in range(3)]
        key = tuple((ranks[0][c[0]], ranks[1][c[1]], ranks[2][c[2]]) for c in coords)
        return self._geom_index.setdefault(key, len(self._geom_index))

    def device_buffers(self):
        return self._buffers('ramp_env_buffers')

    def _buffers(self, fn):
        import ctypes as C

        class _Buf(C.Structure):
            _fields_ = ([(n, C.c_void_p) for n in ('actions', 'reward', 'done', 'queued_model', 'obs_dynamic', 'action_mask', 'busy', 'template_id')]
                        + [(n, C.c_int32) for n in ('n_episodes', 'n_actions', 'n_models')])
        b = _Buf()
        getattr(self.eng._L, fn).restype = C.c_int
        getattr(self.eng._L, fn).argtypes = [C.c_void_p, C.c_void_p]
        _engine._check(getattr(self.eng._L, fn)(self.eng._h, C.byref(b)))
        return {n: getattr(b, n) for n, _ in _Buf._fields_}

    @property
    def queued(self):
        return self.eng.episode_state()[:, EP['queued_job']].astype(np.int64)

    @property
    def last_stats(self):
        import ctypes as C
        out = np.zeros((self.B, _engine.STEP_STATS_LEN), dtype=np.float64)
        self.eng._L.ramp_get_last_step_stats.restype = C.c_int
        self.eng._L.ramp_get_last_step_stats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _engine._check(self.eng._L.ramp_get_last_step_stats(self.eng._h, out.ctypes.data, None))
        return out

    def _read(self):
        _engine._check(self.eng._L.ramp_env_read(self.eng._h, self._reward.ctypes.data, self._done.ctypes.data, self._qmodel.ctypes.data,
                                                 self._obs_dyn.ctypes.data, self._mask.ctypes.data))
        self.done = self._done.astype(bool)
        return {'model': self._qmodel.copy(), 'graph_features_dynamic': self._obs_dyn.copy(), 'action_set': self.action_set,
                'action_mask': self._mask.astype(np.int16), 'done': self.done.copy()}

    def reset(self):
        self.arrivals = self._draw_streams()
        macc = self.macc_override if self.macc_override is not None else np.full((self.B, self.J), np.nan)
        model_of = np.ascontiguousarray(self.model_of, dtype=np.int32)
        frac = np.ascontiguousarray(self.frac, dtype=np.float64)
        macc = np.ascontiguousarray(macc, dtype=np.float64)
        arr = np.ascontiguousarray(self.arrivals, dtype=_engine.ARRIVAL_DTYPE)
        self._keep_reset = (model_of, frac, macc, arr)
        _engine._check(self.eng._L.ramp_env_reset(self.eng._h, model_of.ctypes.data, frac.ctypes.data, macc.ctypes.data, arr.ctypes.data))
        self.eng.n_jobs = self.J
        self.step_counter = 0
        return self._read()

    def step(self, actions=None):
        """actions: int array [B] on the host, or None when a device-resident policy already wrote ramp_env_buffers_t.actions."""
        import ctypes as C
        L, h = self.eng._L, self.eng._h
        n_need = C.c_int32(0)
        a_ptr = None
        if actions is not None:
            self._actions_pinned[:] = np.asarray(actions).reshape(self.B)
            actions = self._actions_pinned
            a_ptr = actions.ctypes.data
        if self._device_decides_everything:
            # no episode can need the host's placer: nothing to wait for between the decision and the cluster step (an invalid
            # action still raises, at the read below)
            _engine._check(L.ramp_env_decide(h, a_ptr, None, None))
        else:
            _engine._check(L.ramp_env_decide(h, a_ptr, C.byref(n_need), self._need.ctypes.data))
            if n_need.value > 0:
                self._decide_on_host(self._need[:n_need.value].copy(), actions)
        _engine._check(L.ramp_env_advance(h))
        obs = self._read()                                     # ONE synchronisation per step; raises simulation errors too
        self.step_counter += 1
        return obs, self._reward.copy(), self.done.copy(), {}

    def step_device(self):
        """One RampJobPartitioningEnvironment.step per episode with the actions a device-resident policy left in
        ``ramp_env_buffers_t.actions`` -- and nothing else: no observation, reward or done flag crosses PCIe (``read()`` fetches them
        when wanted, ``decisions()`` the env-steps every episode has taken).  When every (model, degree) the action set allows is
        decided by the device tables (``prewarm()`` registered every block geometry, no model splits its ops unevenly) the call does
        not even synchronise."""
        import ctypes as C
        L, h = self.eng._L, self.eng._h
        if self._device_decides_everything:
            _engine._check(L.ramp_env_decide(h, None, None, None))
        else:
            n_need = C.c_int32(0)
            _engine._check(L.ramp_env_decide(h, None, C.byref(n_need), self._need.ctypes.data))
            if n_need.value > 0:
                self._decide_on_host(self._need[:n_need.value].copy(), None)
        _engine._check(L.ramp_env_advance(h))
        self.step_counter += 1

    def read(self):
        """Host copies of what the last step left on the device: (obs, reward, done)."""
        obs = self._read()
        self.eng.check_status()
        return obs, self._reward.copy(), self.done.copy()

    def decisions(self):
        """[B] env-steps every episode has taken since reset()."""
        import ctypes as C
        out = np.zeros(self.B, dtype=np.int32)
        L = self.eng._L
        L.ramp_env_read_state.restype = C.c_int
        L.ramp_env_read_state.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _engine._check(L.ramp_env_read_state(self.eng._h, None, None, out.ctypes.data))
        return out

    def record_steps(self, horizon: int):
        """Keeps EvalLoop's results['step_stats'] on the device from now on (ramp_env_steplog_begin): every env-step's row, action
        and reward for up to `horizon` env-steps per episode, written by each step without a synchronisation.  0 stops recording and
        frees the record.  ``recorded_steps()`` reads it back."""
        import ctypes as C
        L = self.eng._L
        L.ramp_env_steplog_begin.restype = C.c_int
        L.ramp_env_steplog_begin.argtypes = [C.c_void_p, C.c_int32]
        _engine._check(L.ramp_env_steplog_begin(self.eng._h, int(horizon)))
        self._log_horizon = int(horizon)

    def recorded_steps(self):
        """EvalLoop's results['step_stats'] (loops/eval_loop.py:44-100) of every episode since ``record_steps``: ``action``,
        ``reward`` and the ``engine.ENV_STEP_STATS`` keys, each a list of B arrays with one entry per env-step the episode took.
        One copy back."""
        import ctypes as C
        H, B, K = getattr(self, '_log_horizon', 0), self.B, _engine.ENV_STEP_STATS_LEN
        if H <= 0:
            raise Exception('no env-step record: call record_steps(horizon) first')
        stats, rewards = np.zeros((H, K, B)), np.zeros((H, B))
        actions, n = np.zeros((H, B), dtype=np.int32), np.zeros(B, dtype=np.int32)
        L = self.eng._L
        L.ramp_env_steplog_read.restype = C.c_int
        L.ramp_env_steplog_read.argtypes = [C.c_void_p, C.c_int32] + [C.c_void_p] * 4
        _engine._check(L.ramp_env_steplog_read(self.eng._h, H, stats.ctypes.data, actions.ctypes.data, rewards.ctypes.data, n.ctypes.data))
        if (n > H).any():
            raise Exception(f'an episode took {int(n.max())} env-steps, the record holds {H}')
        cols = _engine.env_step_columns(stats.transpose(2, 0, 1))       # [B][H] per key
        out = {'action': [actions[:n[b], b].astype(np.int64) for b in range(B)], 'reward': [rewards[:n[b], b].copy() for b in range(B)]}
        for k in _engine.ENV_STEP_STATS:
            out[k] = [cols[k][b, :n[b]] for b in range(B)]
        return out

    def _episode_tables(self):
        import ctypes as C
        job_template = np.zeros((self.B, self.J), dtype=np.int32)
        ret = np.zeros(self.B, dtype=np.float64)
        L = self.eng._L
        L.ramp_env_read_episode.restype = C.c_int
        L.ramp_env_read_episode.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _engine._check(L.ramp_env_read_episode(self.eng._h, job_template.ctypes.data, ret.ctypes.data))
        return job_template, ret

    def _decide_on_host(self, episodes, actions):
        """Episodes the device tables could not decide: full native placer + expansion, then patch the rows (and remember the
        template of the geometry so that the device decides it next time)."""
        import ctypes as C
        L, h = self.eng._L, self.eng._h
        nw = self.n_words
        busy = np.zeros((self.B, nw), dtype=np.uint64)
        dev_actions = np.zeros(self.B, dtype=np.int32)
        L.ramp_env_read_state.restype = C.c_int
        L.ramp_env_read_state.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _engine._check(L.ramp_env_read_state(h, busy.ctypes.data, dev_actions.ctypes.data, None))
        if actions is None:
            actions = dev_actions
        ep = self.eng.episode_state()
        q = ep[:, EP['queued_job']].astype(np.int64)
        keys = {}
        for b in episodes:
            keys.setdefault((int(self.model_of[b, q[b]]), int(actions[b])) + tuple(int(x) for x in busy[b]), []).append(int(b))
        by_md = {}
        for key in keys:
            if key not in self._placement_cache:
                by_md.setdefault(key[:2], []).append(key)
        for (m, d), ks in by_md.items():
            self._place_many(m, d, np.array([k[2:] for k in ks], dtype=np.uint64).reshape(-1, nw))
        mounts = self._t_mount
        for key, bs in keys.items():
            tid, words = self._placement_cache[key]
            mask = np.array(words, dtype=np.uint64)
            mt = np.array(mounts[tid] if tid >= 0 else (0.0,) * 6, dtype=np.float64)
            m, d = key[0], key[1]
            if tid >= 0 and self._uniform[m, d]:
                coords = [self._servers[i] for i in range(self.W) if (words[i >> 6] >> (i & 63)) & 1]
                gkey = self._geometry(coords)
                if gkey < self._n_geoms and (m, d, gkey) not in self._table_set:
                    _engine._check(L.ramp_env_set_template(h, m, d, gkey, tid, mt.ctypes.data))
                    self._table_set.add((m, d, gkey))
            elif tid >= 0 and self.place_on_device:
                coords = [self._servers[i] for i in range(self.W) if (words[i >> 6] >> (i & 63)) & 1]
                cm = self._canonical_mask(coords)
                if (m, d, cm) not in self._geom_mask_set:
                    cw = np.array(cm, dtype=np.uint64)
                    _engine._check(L.ramp_env_set_geometry_template(h, m, d, cw.ctypes.data, tid, mt.ctypes.data))
                    self._geom_mask_set.add((m, d, cm))
            for b in bs:
                _engine._check(L.ramp_env_patch(h, b, tid, mask.ctypes.data, mt.ctypes.data))

