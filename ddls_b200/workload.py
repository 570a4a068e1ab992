"""Scripted synthetic rollouts at BASELINE.json's sizes (no reference, no dataset needed).

A *workload* is: a RAMP shape, a set of lowered-job templates (one per (model, partition degree)), and for
each of B episodes a script of L agent decisions (one per arriving job): which template to mount (or -1 =
do not place, RJPE action 0) with that job's mount scalars, plus the arrival stream.  The decisions are
produced by a documented stand-in for the reference's agents (which stay Python and are not part of the
hot path): a random partition-degree policy (the role PAC-ML's GNN policy plays in BASELINE.json config 3)
and an aligned first-fit block allocator that respects RAMP rule 1 (one job per worker, ramp_rules.py:1-40).
The allocator needs to know when jobs finish, so the generator runs a small host-side timeline using each
template's job completion time (computed once by whoever builds the workload -- the CUDA engine in the
product path, the oracle in CPU tests).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, List, Sequence

import numpy as np

from . import synth
from .lowered import LoweredJob
from .template_builder import RampShape, build_template

ARRIVAL_DTYPE = np.dtype([('interarrival', np.float64), ('orig_op_mem', np.float64), ('orig_dep_size', np.float64)])
ACTION_DTYPE = np.dtype([('max_acceptable_jct', np.float64), ('part_op_mem', np.float64), ('part_dep_size', np.float64),
                         ('flow_size', np.float64), ('n_mounted_workers', np.int32), ('n_mounted_channels', np.int32),
                         ('template_id', np.int32), ('flags', np.int32)])

CONFIGS = {
    # BASELINE.json configs[0]: 8-worker RAMP, chain DAG, random partition degree
    'cfg1-chain-8w': dict(shape=(2, 2, 2), graphs=[('chain', {})], degrees=(2, 4, 8), n_episodes=1),
    # configs[1]: 256 episodes, 32-worker RAMP, ResNet-50-like
    'cfg2-resnet50-32w': dict(shape=(4, 4, 2), graphs=[('resnet', {})], degrees=(2, 4, 8, 16), n_episodes=256),
    # configs[2] (the configuration BASELINE.json's metric / north_star target is quoted on)
    'cfg3-resnet50-64w': dict(shape=(4, 4, 4), graphs=[('resnet', {})], degrees=(2, 4, 8, 16), n_episodes=4096),
    # configs[3]: 256-worker RAMP, BERT-base-like
    'cfg4-bert-256w': dict(shape=(8, 8, 4), graphs=[('bert', {})], degrees=(2, 4, 8, 16), n_episodes=4096),
    # configs[4]: 128-worker RAMP, ResNet-50 + GPT-2-small mix, exponential inter-arrivals
    'cfg5-mix-128w': dict(shape=(8, 4, 4), graphs=[('resnet', {}), ('gpt2', {})], degrees=(2, 4, 8, 16), n_episodes=16384,
                          exponential=True),
}


def scripted_job_totals(g: synth.ForwardGraph):
    """(orig_op_mem, orig_dep_size) the scripted arrival rows carry for a job of graph g: twice the ops' memory (activation +
    parameters), and every dep of the mirrored job sized by its source op's memory.  These rows are an input of the workload
    (the load rate and the demand_* sums of every step read them), fixed so that every version of the simulator is measured on
    the same workload and its outputs stay comparable; both arms read the same rows.  They are not the reference's job totals
    (``template_builder.original_job_totals`` is, and the batched environments use it): the dep sizes there are activations only."""
    mem = [a + p for a, p in zip(g.act, g.par)]
    dep = 0.0
    for (u, v) in g.edges:
        dep += mem[u - 1]            # forward edge: the source op
        dep += mem[v - 1]            # mirrored backward edge 2n-(v-1) -> 2n-(u-1): its source mirrors v
    dep += mem[g.n - 1]              # join edge n -> n+1
    return 2.0 * sum(mem), dep


def make_graph(kind, **kw):
    if kind == 'chain':
        return synth.chain_graph(**kw)
    if kind == 'resnet':
        return synth.resnet_like_graph(**kw)
    if kind == 'bert':
        return synth.transformer_like_graph(n_layers=12, name='bert_base_like', seed=2, **kw)
    if kind == 'gpt2':
        return synth.transformer_like_graph(n_layers=12, name='gpt2_small_like', seed=5, gpt=True, **kw)
    if kind == 'residual54':
        return synth.residual_small_graph(**kw)
    raise Exception(f'unknown graph kind {kind}')


@dataclass
class Workload:
    name: str
    shape: RampShape
    templates: List[LoweredJob]
    template_model: List[int]
    template_degree: List[int]
    n_episodes: int
    n_steps: int                       # L: agent decisions (= arriving jobs) per episode
    arrivals: np.ndarray = None        # [B, L] ARRIVAL_DTYPE
    actions: np.ndarray = None         # [L, B] ACTION_DTYPE (template_id indexes `templates`)
    max_sim_time: float = float('inf')
    meta: dict = field(default_factory=dict)


def reference_template(g, degree, shape: RampShape, quantum=0.01, num_training_steps=50, model_id=0):
    """The lowered job the reference's own pipeline produces for ``g`` at max partition degree ``degree`` on an EMPTY cluster:
    RampFirstFitOpPlacer's block (ramp_first_fit_place), then OpPartition / update_dep_run_times (collectives) / SRPT schedulers /
    FirstFitDepPlacer (ramp_expand_template, run_times='reference').  Equal to the reference-lowered job in every array but the
    hash-ordered priority ties (tests/test_expand_native.py); needs libramp_b200.so (host-only code, no GPU)."""
    import math
    from .expand import expand_template
    from .placer import first_fit_place_native
    splits = [int(max(1, min(math.ceil(math.ceil(c / quantum) / 2) * 2, degree))) for c in g.fwd]      # RJPE:332-343
    servers = [(c, r, s) for c in range(shape.c) for r in range(shape.r) for s in range(shape.s)]
    where = first_fit_place_native(g.n, [a + p for a, p in zip(g.act, g.par)], g.edges, splits,
                                   {sv: 80e9 for sv in servers}, {sv: False for sv in servers}, (shape.c, shape.r, shape.s))
    if where is None:
        raise Exception(f'{g.name} does not fit an empty {shape.c}x{shape.r}x{shape.s} cluster at degree {degree}')
    return expand_template(g, degree, shape, quantum=quantum, num_training_steps=num_training_steps, model_id=model_id,
                           run_times='reference', coords=sorted(set(where.values())))


def build_templates(config: str, quantum=0.01, num_training_steps=50, run_times='one_to_one'):
    """run_times='one_to_one': template_builder's aligned blocks and one-to-one transfer times (pure Python, no library needed);
    'reference': the reference pipeline's lowered jobs on an empty cluster (reference_template)."""
    cfg = CONFIGS[config]
    shape = RampShape(*cfg['shape'])
    templates, t_model, t_degree, graphs = [], [], [], []
    for m, (kind, kw) in enumerate(cfg['graphs']):
        g = make_graph(kind, **kw)
        graphs.append(g)
        for d in cfg['degrees']:
            if d > shape.n_workers:
                continue
            if run_times == 'reference':
                templates.append(reference_template(g, d, shape, quantum=quantum, num_training_steps=num_training_steps, model_id=m))
            else:
                templates.append(build_template(g, d, shape, block_start=0, quantum=quantum,
                                                num_training_steps=num_training_steps, model_id=m))
            t_model.append(m)
            t_degree.append(d)
    return cfg, shape, graphs, templates, t_model, t_degree


def generate(config: str, jct_of_template: Callable[[Sequence[LoweredJob]], Sequence[float]], n_episodes: int = None,
             n_steps: int = 8, seed: int = 0, interarrival: float = 1000.0, run_times: str = 'one_to_one') -> Workload:
    """Builds the templates and B scripted episodes of L decisions each.

    jct_of_template(templates) -> lookahead job completion time per template (from the engine or the oracle).
    """
    cfg, shape, graphs, templates, t_model, t_degree = build_templates(config, run_times=run_times)
    B = n_episodes or cfg['n_episodes']
    L = n_steps
    rng = np.random.default_rng(seed)
    jct = np.asarray(jct_of_template(templates), dtype=np.float64)
    n_models = len(graphs)
    totals = [scripted_job_totals(g) for g in graphs]
    by_model = [[t for t in range(len(templates)) if t_model[t] == m] for m in range(n_models)]

    # arrival streams (JobsGenerator stand-in): model per job, inter-arrival gaps, max-acceptable fraction
    model_of = rng.integers(0, n_models, size=(B, L))
    if cfg.get('exponential'):
        gaps = rng.exponential(interarrival, size=(B, L))
    else:
        gaps = np.full((B, L), float(interarrival))
    gaps[:, L - 1] = np.inf                                   # no job after the last one (jobs_generator.py:270-272)
    frac = np.round(rng.uniform(0.1, 1.0, size=(B, L)), 2)    # Uniform(0.1, 1, decimals=2) heuristic_config.yaml:115-118
    arrivals = np.zeros((B, L), dtype=ARRIVAL_DTYPE)
    arrivals['interarrival'] = gaps
    arrivals['orig_op_mem'] = np.array([totals[m][0] for m in range(n_models)])[model_of]
    arrivals['orig_dep_size'] = np.array([totals[m][1] for m in range(n_models)])[model_of]

    # agent stand-in: random degree + aligned first-fit block allocation on a host-side timeline
    pick = rng.integers(0, 1 << 30, size=(B, L))
    actions = np.zeros((L, B), dtype=ACTION_DTYPE)
    actions['template_id'] = -1
    n_w = shape.n_workers
    t_arr = np.concatenate([np.zeros((B, 1)), np.cumsum(gaps[:, :-1], axis=1)], axis=1)   # arrival time of job k
    busy_until = np.zeros((B, n_w))                           # per worker: time its current job completes
    for k in range(L):
        now = t_arr[:, k]
        cand = np.array([by_model[m][pick[b, k] % len(by_model[m])] for b, m in enumerate(model_of[:, k])])
        deg = np.array(t_degree)[cand]
        free = busy_until <= (now[:, None] + 1e-7)            # [B, n_w]
        tid = np.full(B, -1, dtype=np.int32)
        for d in sorted(set(deg.tolist())):
            sel = np.nonzero(deg == d)[0]
            if not len(sel):
                continue
            blocks = free[sel].reshape(len(sel), n_w // d, d).all(axis=2)      # aligned blocks of d workers
            has = blocks.any(axis=1)
            first = blocks.argmax(axis=1)
            ok = sel[has]
            tid[ok] = cand[ok]
            macc = frac[ok, k] * np.array([templates[t].seq_time for t in cand[ok]])
            accepted = jct[cand[ok]] <= macc                   # RCE:815: blocked iff jct > max acceptable
            for b, f, acc in zip(ok, first[has], accepted):
                if acc:
                    busy_until[b, f * d:(f + 1) * d] = now[b] + jct[cand[b]]
        placed = tid >= 0
        for t in range(len(templates)):
            m = templates[t].mount
            s = placed & (tid == t)
            if not s.any():
                continue
            actions[k]['max_acceptable_jct'][s] = frac[s, k] * templates[t].seq_time
            actions[k]['part_op_mem'][s] = m.part_op_mem
            actions[k]['part_dep_size'][s] = m.part_dep_size
            actions[k]['flow_size'][s] = m.flow_size
            actions[k]['n_mounted_workers'][s] = m.n_mounted_workers
            actions[k]['n_mounted_channels'][s] = m.n_mounted_channels
        actions[k]['template_id'] = tid
    wl = Workload(name=config, shape=shape, templates=templates, template_model=t_model, template_degree=t_degree,
                  n_episodes=B, n_steps=L, arrivals=arrivals, actions=actions,
                  meta=dict(seed=seed, interarrival=interarrival, degrees=list(cfg['degrees']), run_times=run_times,
                            placed_frac=float((actions['template_id'] >= 0).mean())))
    return wl
