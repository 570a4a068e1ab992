"""The thread-per-lookahead kernel (ddls_b200/csrc/ramp_lookahead_thread.cuh) on both of its routes, against the CPU oracle.

A template's first lookahead ("first launch") may spill its frontiers to HBM, stages its trace in a per-CTA buffer and
computes the utilisation in the epilogue; it then records TemplateHints (ticks, largest ready-op / ready-flow /
ready-non-flow frontiers) and hint_jct.  Every later one ("hinted") trusts those hints: no list leaves shared memory,
the trace is written in place and the utilisation is summed by the ledger lane inside the tick loop.  A hint that
under-states a frontier would write past its shared-memory list without faulting, so the hints are checked against a
model of the frontiers (tests/quotient_model.py) as well as the results against the oracle.

Tests without the gpu mark check the boundary templates on the model alone and run without a GPU.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from conftest import golden_files
from golden_io import Golden
import quotient_model as qm
from ddls_b200.quotient import quotient as native_quotient

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = golden_files()
THREAD_MODES = ['thread', 'thread_unfolded']
MODES = THREAD_MODES + ['warp', 'cta']
OCAP, FASTF, FCAP, NFCAP, WCAP, CCAP = 8, 6, 16, 8, 8, 32    # RAMP_T_* of the normal build
RES_MAX_BYTES = 96 * 1024                                 # ramp_engine.cu res_max_bytes
MODEL_MAX_WORK = 20_000_000                               # (classes + entries) x ticks the Python model is run for


# ---------------------------------------------------------------------------------------------------------------------
# small lowered jobs
def _job(op_cost, op_worker, edges, n_workers, n_channels, num_training_steps=2):
    """edges: (src, dst, run_time, is_flow, channel or None, priority); op priorities follow the op index (first wins)."""
    from ddls_b200.lowered import LoweredJob, MountScalars, NO_CHANNEL
    N = len(op_cost)
    edges = sorted(edges, key=lambda e: e[0])                     # CSR by source (stable: keeps the given dep order)
    row = np.zeros(N + 1, dtype=np.int64)
    for e in edges:
        row[e[0] + 1] += 1
    row = np.cumsum(row)
    n_par = np.zeros(N, dtype=np.int64)
    for e in edges:
        n_par[e[1]] += 1
    return LoweredJob(n_ops=N, n_deps=len(edges), n_workers=n_workers, n_channels=n_channels,
                      num_training_steps=num_training_steps, model_id=0, degree=1,
                      op_cost=np.asarray(op_cost, dtype=np.float64), op_prio=np.arange(N)[::-1].copy(),
                      op_worker=np.asarray(op_worker), op_n_parents=n_par, row_ptr=row,
                      dep_dst=np.array([e[1] for e in edges], dtype=np.int64),
                      dep_run_time=np.array([e[2] for e in edges], dtype=np.float64),
                      dep_prio=np.array([e[5] for e in edges], dtype=np.int64),
                      dep_channel=np.array([NO_CHANNEL if e[4] is None else e[4] for e in edges], dtype=np.int64),
                      dep_is_flow=np.array([e[3] for e in edges], dtype=np.uint8),
                      mount=MountScalars(n_mounted_workers=n_workers)).canonicalise()


def ready_ops_template(k, simple):
    """k source op classes ready at once (distinct costs): one worker, or two (a second worker group)."""
    return _job([1.0 + 0.125 * i for i in range(k)], [0 if simple else i % 2 for i in range(k)], [], 1 if simple else 2, 0)


def ready_flows_template(k, simple):
    """op 0 -> op 1 through k flows of distinct run times: all k ready when op 0 completes.  Non-simple: alternate
    channels (two channel groups)."""
    edges = [(0, 1, 0.5 + 0.25 * i, 1, 0 if simple else i % 2, i) for i in range(k)]
    return _job([1.0, 0.75], [0, 0 if simple else 1], edges, 1 if simple else 2, 1 if simple else 2)


def ready_nonflows_template(k, simple):
    """op 0 -> k children (distinct costs) through non-flow deps: k ready non-flow entries in one tick, and then k
    readied op classes."""
    edges = [(0, 1 + i, 0.0, 0, None, i) for i in range(k)]
    return _job([1.0] + [1.0 + 0.25 * i for i in range(k)], [0] + [0 if simple else i % 2 for i in range(k)], edges,
                1 if simple else 2, 0)


def many_worker_groups_template(n_groups=10):
    """Two ops on each of n_groups workers (> RAMP_T_WCAP): winners by pairwise comparison, then one flow each to a sink."""
    N = 2 * n_groups + 1
    cost = [1.0 + 0.125 * i for i in range(2 * n_groups)] + [0.5]
    worker = [i % n_groups for i in range(2 * n_groups)] + [0]
    edges = [(i, N - 1, 0.25 + 0.125 * i, 1, i % 4, i) for i in range(2 * n_groups)]
    return _job(cost, worker, edges, n_groups, 4)


def channel_groups_template(n_groups):
    """op 0 -> n_groups children, one flow each on its own channel (distinct run times): n_groups channel groups."""
    edges = [(0, 1 + i, 0.5 + 0.25 * i, 1, i, i) for i in range(n_groups)]
    return _job([1.0] + [0.5] * n_groups, [0] + [1] * n_groups, edges, 2, n_groups)


# (name, template, peak field, intended peak, simple)
def boundary_cases():
    cases = []
    for simple in (True, False):
        s = 'simple' if simple else 'general'
        for k in (2, 3, OCAP, OCAP + 1):
            cases.append((f'ops{k}-{s}', ready_ops_template(k, simple), 'max_o', k, simple))
        for k in (FASTF, FASTF + 1, FCAP, FCAP + 1):
            cases.append((f'flows{k}-{s}', ready_flows_template(k, simple), 'max_f', k, simple))
        for k in (NFCAP, NFCAP + 1):
            cases.append((f'nonflows{k}-{s}', ready_nonflows_template(k, simple), 'max_nf', k, simple))
    cases.append(('workers10', many_worker_groups_template(10), 'max_o', 20, False))
    return cases


BOUNDARY = boundary_cases()
BOUNDARY_IDS = [c[0] for c in BOUNDARY]


def model_peaks(job, mode):
    q = native_quotient(job) if mode == 'thread' else qm.identity_quotient(job)
    return q, qm.run_lookahead_quotient(q)


def resident_rule(job, q):
    """ramp_engine.cu build_resident_blob's eligibility, restated: the quotient fits the 96 KB blob, its counters 16 bits,
    it has at most RAMP_T_CCAP channel groups, and a dep word's key + one bit per channel group fit 32 bits."""
    N, E = q.n_ops, q.n_deps
    if N < 1 or not q.masks_valid or q.n_channels > CCAP:
        return False
    bits = lambda v: max(1, int(v).bit_length())
    in_total = np.bincount(q.dep_dst, weights=q.dep_inc, minlength=N) if E else np.zeros(N)
    if (q.op_weight > 0xFFFF).any() or (in_total > 0xFFFF).any():
        return False
    kbits = bits(len(np.unique(q.dep_key)) + 1)
    if kbits + max(q.n_channels, 1) > 32 or 1 + bits(max(q.dep_inc.max() if E else 1, 1)) + bits(N) > 32:
        return False
    a16 = lambda v: (v + 15) // 16 * 16
    n_src = int((np.bincount(q.dep_dst, minlength=N) == 0).sum()) if E else N
    return 96 + a16(N * 16) + a16(N * 8) + a16(N * 4) + a16(max(E, 1) * 16) + a16(max(n_src, 1) * 4) <= RES_MAX_BYTES


# ---------------------------------------------------------------------------------------------------------------------
# model only (no GPU)
@pytest.mark.parametrize('name,job,field,peak,simple', BOUNDARY, ids=BOUNDARY_IDS)
def test_boundary_template_reaches_its_peak(name, job, field, peak, simple):
    """Each boundary template's frontier peak lands exactly where it is meant to, on the quotient the kernel runs."""
    for mode in THREAD_MODES:
        q, m = model_peaks(job, mode)
        assert m['finished']
        assert m[field] == peak, (mode, m)
        assert ((q.n_workers == 1) and (q.n_channels <= 1)) == simple, (mode, q.n_workers, q.n_channels)
        assert resident_rule(job, q)
    if name == 'workers10':
        assert native_quotient(job).n_workers > WCAP


def test_model_peaks_match_the_oracle_traces(oracle_lib):
    """The frontier model is the kernels' tick loop: its trace on every boundary template is the oracle's."""
    for name, job, *_ in BOUNDARY:
        o = oracle_lib.run_lookahead(job)
        for mode in THREAD_MODES:
            _, m = model_peaks(job, mode)
            assert m['n_ticks'] == o['n_ticks'] and m['jct'] == o['jct'], (name, mode)
            np.testing.assert_array_equal(m['trace_tick'], o['trace_tick'])
            np.testing.assert_array_equal(m['trace_n_active'], o['trace_n_active'])


@pytest.mark.parametrize('n_groups', [32, 40])
def test_32_channel_groups_are_never_resident(n_groups):
    """A resident template has at most RAMP_T_CCAP = 32 channel groups, the size of the thread kernel's per-channel-group
    winner table, which is its only channel-winner path.  A resident dep word also holds the key and one bit per channel
    group in 32 bits, so in fact 32 groups are already too many."""
    job = channel_groups_template(n_groups)
    q = native_quotient(job)
    assert q.n_channels == n_groups
    assert not resident_rule(job, q)


# which golden templates the 'thread' / 'thread_unfolded' modes really run on the thread kernel (the rest go to the warp /
# CTA kernels): {file: (resident in thread mode, resident in thread_unfolded mode)}, template indices
#   Not resident: quotient blobs over 96 KB (e.g. resnet64_deg4_full: 6,673 entries x 16 B), or key bits + channel groups
#   over 32 (e.g. chain8 templates 0-2 and 14: 49 channel groups).  Their 'thread' parity runs test the warp / CTA kernels.
RESIDENT = {
    'bert256_shard.npz': ([], []),
    'chain8.npz': ([3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 15], [3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 15]),
    'chain8_busy.npz': ([0, 1, 2, 3, 4, 5, 6, 7], [0, 1, 2, 3, 4, 5, 6, 7]),
    'chain8_maxtime.npz': ([0, 1, 2, 3], [0, 1, 2, 3]),
    'mix128_exp.npz': ([0, 1, 2, 3, 4, 5], [0, 1, 4, 5]),
    'mixed16.npz': ([1, 2, 5, 8, 10, 11], [1, 2, 5, 8, 10, 11]),
    'mixed64_busy.npz': ([1, 2, 3, 4, 7, 11, 12, 15, 16, 17, 19, 21, 22], [1, 2, 3, 4, 11, 15, 19, 21]),
    'res16_flood.npz': ([0, 1, 2, 3, 4, 5], [0, 1, 2, 3, 4, 5]),
    'residual32_deg16.npz': ([], []),
    'residual8_deg4.npz': ([0, 1, 2, 3], [0, 1, 2, 3]),
    'resnet32_cfg2.npz': ([], []),
    'resnet64_deg16_full.npz': ([], []),
    'resnet64_deg2_full.npz': ([0], [0]),
    'resnet64_deg4_full.npz': ([], []),
    'resnet64_deg8_full.npz': ([], []),
    'tfm32_acceptable.npz': ([0, 2, 3, 4, 5], [0, 2, 3, 4, 5]),
}
# the 60 random templates and the 4 baseline-sized ones (degrees 2, 4, 8, 16) of _random_and_baseline
RESIDENT_RANDOM = {'thread': (32, [True, True, True, True]), 'thread_unfolded': (32, [True, False, False, False])}


def _resident_sets(g):
    out = []
    for mode in THREAD_MODES:
        out.append([k for k, t in enumerate(g.templates)
                    if resident_rule(t, native_quotient(t) if mode == 'thread' else qm.identity_quotient(t))])
    return tuple(out)


@pytest.mark.parametrize('fname', FILES)
def test_resident_golden_templates_are_pinned(fname):
    """The set of golden templates the thread kernel simulates cannot shrink unnoticed."""
    assert _resident_sets(Golden(fname)) == RESIDENT[fname]


@pytest.mark.parametrize('mode', THREAD_MODES)
def test_resident_random_templates_are_pinned(mode):
    ts = _random_and_baseline()
    r = [resident_rule(t, native_quotient(t) if mode == 'thread' else qm.identity_quotient(t)) for t in ts]
    assert (sum(r[:60]), r[60:]) == RESIDENT_RANDOM[mode]


# ---------------------------------------------------------------------------------------------------------------------
# GPU
@pytest.fixture(scope='module')
def eng_mod():
    import torch
    assert torch.cuda.is_available(), 'these tests need a CUDA device'
    from ddls_b200 import engine
    engine.load_library()
    return engine


def _engine(eng_mod, mode, **kw):
    os.environ['RAMP_LOOKAHEAD_MODE'] = mode
    try:
        return eng_mod.RampEngine(**kw)
    finally:
        os.environ.pop('RAMP_LOOKAHEAD_MODE', None)


def _assert_equal_oracle(res, tn, tt, k, o):
    assert res['status'][k] == o['status'] and res['n_ticks'][k] == o['n_ticks'], k
    np.testing.assert_array_equal(tn[k, :o['n_ticks']], o['trace_n_active'])
    np.testing.assert_array_equal(tt[k, :o['n_ticks']], o['trace_tick'])
    if o['status'] == 0:
        assert res['jct'][k] == o['jct'] and res['comm'][k] == o['comm'] and res['comp'][k] == o['comp'], k


def _check_hints(info, job, o, mode):
    """After a first launch: the hints hold the oracle's tick count and jct bit for bit, and frontiers no smaller than the
    model's peaks (an under-statement would overrun a shared-memory list on the hinted route) -- equal, in fact."""
    if o['status'] != 0:
        assert info['n_ticks'] == 0 and info['hint_jct'] == 0.0
        return
    assert info['n_ticks'] == o['n_ticks'] and info['hint_jct'] == o['jct']
    q = native_quotient(job) if mode == 'thread' else qm.identity_quotient(job)
    if (q.n_ops + q.n_deps) * o['n_ticks'] > MODEL_MAX_WORK:
        return
    m = qm.run_lookahead_quotient(q)
    assert (info['max_o'], info['max_f'], info['max_nf']) == (m['max_o'], m['max_f'], m['max_nf'])


@pytest.mark.gpu
@pytest.mark.parametrize('mode', THREAD_MODES)
@pytest.mark.parametrize('fname', FILES)
def test_golden_hints_and_residency(fname, mode, eng_mod, oracle_lib):
    """Which golden templates run on the thread kernel (pinned above), and what their first launch records."""
    g = Golden(fname)
    eng = _engine(eng_mod, mode, n_episodes=1, n_cluster_workers=g.n_cluster_workers, max_jobs=1, trace_cap=1 << 16)
    tids = [eng.register_template(t) for t in g.templates]
    eng.run_lookaheads(np.array(tids, dtype=np.int32))
    want = RESIDENT[fname][THREAD_MODES.index(mode)]
    for k, t in enumerate(g.templates):
        info = eng.template_info(tids[k])
        assert (info['size_class'] == 2) == (k in want), k
        if info['size_class'] == 2:
            _check_hints(info, t, oracle_lib.run_lookahead(t), mode)
    eng.close()


def _random_and_baseline():
    from ddls_b200 import synth
    from ddls_b200.template_builder import RampShape, build_template, random_dag_template
    rng = np.random.default_rng(1234)
    ts = [random_dag_template(rng, int(n), n_workers=int(w)) for n, w in
          zip(rng.integers(2, 400, size=60), rng.integers(1, 9, size=60))]
    ts += [build_template(synth.resnet_like_graph(), d, RampShape(4, 4, 4)) for d in (2, 4, 8, 16)]
    return ts


@pytest.mark.gpu
@pytest.mark.parametrize('mode', THREAD_MODES)
def test_random_and_baseline_hints(mode, eng_mod, oracle_lib):
    ts = _random_and_baseline()
    eng = _engine(eng_mod, mode, n_episodes=1, n_cluster_workers=64, max_jobs=1, trace_cap=1 << 16)
    tids = [eng.register_template(t) for t in ts]
    eng.run_lookaheads(np.array(tids, dtype=np.int32))
    for k, t in enumerate(ts):
        info = eng.template_info(tids[k])
        q = native_quotient(t) if mode == 'thread' else qm.identity_quotient(t)
        assert (info['size_class'] == 2) == resident_rule(t, q), k
        if info['size_class'] == 2:
            _check_hints(info, t, oracle_lib.run_lookahead(t), mode)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize('launch', ['first', 'hinted'])
@pytest.mark.parametrize('mode', THREAD_MODES)
def test_boundary_templates_vs_oracle(mode, launch, eng_mod, oracle_lib):
    """Every capacity boundary, first launch and hinted: results and traces equal the oracle's, the hints equal the
    model's peaks, and the hinted launch took the shared-memory-only route exactly when the peaks fit."""
    ts = [c[1] for c in BOUNDARY]
    eng = _engine(eng_mod, mode, n_episodes=1, n_cluster_workers=64, max_jobs=1, trace_cap=4096)
    tids = np.array([eng.register_template(t) for t in ts], dtype=np.int32)
    ids = np.repeat(tids, 3)
    if launch == 'hinted':
        eng.run_lookaheads(ids)
    res, _, tn, tt = eng.run_lookaheads(ids, want_trace=True)
    for k, (name, t, field, peak, _) in enumerate(BOUNDARY):
        o = oracle_lib.run_lookahead(t)
        for r in range(3):
            _assert_equal_oracle(res, tn, tt, 3 * k + r, o)
        info = eng.template_info(int(tids[k]))
        assert info['size_class'] == 2, name
        _check_hints(info, t, o, mode)
        assert info[field] == peak, name
    eng.close()


@pytest.mark.gpu
def test_32_channel_groups_run_elsewhere(eng_mod, oracle_lib):
    t = channel_groups_template(32)
    eng = _engine(eng_mod, 'thread', n_episodes=1, n_cluster_workers=64, max_jobs=1, trace_cap=4096)
    tid = eng.register_template(t)
    assert eng.template_info(tid)['size_class'] != 2
    res, _, tn, tt = eng.run_lookaheads(np.full(2, tid, dtype=np.int32), want_trace=True)
    o = oracle_lib.run_lookahead(t)
    _assert_equal_oracle(res, tn, tt, 0, o)
    _assert_equal_oracle(res, tn, tt, 1, o)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize('launch', ['first', 'hinted'])
@pytest.mark.parametrize('mode', THREAD_MODES)
def test_many_chunks_of_one_template_per_launch(mode, launch, eng_mod, oracle_lib):
    """One template 1, 31, 32, 33 and 65 times in one launch, interleaved with others: full and partial chunks, several
    chunks of a template in one launch (some may read the hints another CTA records meanwhile), and a zero-jct job."""
    from ddls_b200 import synth
    from ddls_b200.template_builder import RampShape, build_template
    from test_gpu_parity import zero_jct_template
    g = synth.resnet_like_graph(n_blocks=4, name='res4')
    ts = [build_template(g, d, RampShape(4, 4, 4)) for d in (2, 4, 8, 16, 1)] + [zero_jct_template()]
    counts = [1, 31, 32, 33, 65, 7]
    eng = _engine(eng_mod, mode, n_episodes=1, n_cluster_workers=64, max_jobs=1, trace_cap=4096)
    tids = [eng.register_template(t) for t in ts]
    ids = np.concatenate([np.full(c, tids[k], dtype=np.int32) for k, c in enumerate(counts)])
    ids = ids[np.random.default_rng(3).permutation(len(ids))]
    if launch == 'hinted':
        eng.run_lookaheads(ids)
    res, _, tn, tt = eng.run_lookaheads(ids, want_trace=True)
    want = {tid: oracle_lib.run_lookahead(t) for tid, t in zip(tids, ts)}
    assert want[tids[-1]]['jct'] == 0.0
    for k in range(len(ids)):
        _assert_equal_oracle(res, tn, tt, k, want[int(ids[k])])
    for tid, t in zip(tids, ts):
        info = eng.template_info(tid)
        q = native_quotient(t) if mode == 'thread' else qm.identity_quotient(t)
        assert (info['size_class'] == 2) == resident_rule(t, q)
        if info['size_class'] == 2:
            _check_hints(info, t, want[tid], mode)
    if mode == 'thread':
        assert all(eng.template_info(tid)['size_class'] == 2 for tid in tids)
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize('launch', ['first', 'hinted'])
@pytest.mark.parametrize('mode', MODES)
def test_trace_capacity_boundary(mode, launch, eng_mod, oracle_lib):
    """A lookahead of T ticks fits trace_cap T and T + 1 exactly; trace_cap T - 1 is RAMP_ST_TRACE_OVERFLOW, which the step
    path raises."""
    from ddls_b200 import synth
    from ddls_b200.engine import action_row
    from ddls_b200.template_builder import RampShape, build_template
    t = build_template(synth.resnet_like_graph(n_blocks=4, name='res4'), 4, RampShape(4, 4, 4))
    o = oracle_lib.run_lookahead(t)
    T = o['n_ticks']
    for cap in (T - 1, T, T + 1):
        eng = _engine(eng_mod, mode, n_episodes=1, n_cluster_workers=64, max_jobs=2, trace_cap=cap)
        tid = eng.register_template(t)
        ids = np.full(3, tid, dtype=np.int32)
        if launch == 'hinted':
            eng.run_lookaheads(ids)
        res, _, tn, tt = eng.run_lookaheads(ids, want_trace=True)
        if cap < T:
            assert (res['status'] == 2).all(), (cap, res)
            assert eng.template_info(tid)['n_ticks'] == 0           # an overflowing lookahead records no hints
        else:
            for k in range(3):
                _assert_equal_oracle(res, tn, tt, k, o)
        arr = np.zeros((1, 2), dtype=eng_mod.ARRIVAL_DTYPE)
        arr['interarrival'] = [[1.0, np.inf]]
        eng.reset(arr)
        a = eng.make_actions()
        action_row(a, 0, tid, t.mount)
        eng.step(a)
        if cap < T:
            with pytest.raises(Exception, match='trace_cap'):
                eng.check_status()
        else:
            eng.check_status()
            la = eng.last_lookahead(0)
            assert la['status'] == 0 and la['jct'] == o['jct'] and la['n_ticks'] == T
            np.testing.assert_array_equal(la['trace_tick'], o['trace_tick'])
        eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize('memo_mode', [1, 2])
@pytest.mark.parametrize('fname', FILES)
def test_step_path_utilisation_vs_oracle(fname, memo_mode, eng_mod, oracle_lib):
    """Golden arrival streams replayed for B = 40 episodes (two chunks of a template per launch), each mounting the step's
    job on its own number of workers.  Memo off: every mount runs a fresh lookahead -- a template's first step takes the
    first-launch route, later ones the hinted route (utilisation summed in the tick loop, trace written in place).  Exact
    memo: one episode runs the lookahead, the others hit it with another worker count and the step kernel recomputes the
    utilisation from the stored trace.  Every mounted job's jct / comm / comp and utilisation, and every mount's trace,
    equal the oracle's bit for bit.
    Trace pool: memo off stores B x (sum over mounting steps of the template's ticks) entries, at most 246,920 for these
    fixtures -- far below the pool's 4 Mi entries (it is only reset by ramp_reset)."""
    from ddls_b200.engine import EP, JS_COMPLETED, JS_RUNNING, action_row
    g = Golden(fname)
    B = 40
    arr = g.arrivals()
    eng = eng_mod.RampEngine(n_episodes=B, n_cluster_workers=g.n_cluster_workers, max_jobs=len(arr), memo_mode=memo_mode,
                             max_simulation_run_time=g.max_sim_time, trace_cap=1 << 16)
    tids = [eng.register_template(t) for t in g.templates]
    want = {}
    pool_entries = 0
    eng.reset(np.stack([arr] * B))
    mounted = {}                                   # (episode, job idx) -> (template, n_mounted_workers)
    for s in range(g.n_steps):
        job = g.step_job(s)
        a = eng.make_actions()
        if job is not None:
            k = int(g.d['step_tid'][s])
            if k not in want:
                want[k] = oracle_lib.run_lookahead(g.templates[k])
            pool_entries += B * want[k]['n_ticks']
            queued = eng.episode_state()[:, EP['queued_job']].astype(int)
            for b in range(B):
                action_row(a, b, tids[k], job.mount)
                a['n_mounted_workers'][b] = max(1, job.mount.n_mounted_workers - (b % 4))
                mounted[(b, queued[b])] = (k, int(a['n_mounted_workers'][b]))
        eng.step(a)
        eng.check_status()
        if job is not None:
            o = want[k]
            for b in range(B):
                la = eng.last_lookahead(b)
                assert la['status'] == 0 and la['n_ticks'] == o['n_ticks'] and la['jct'] == o['jct'], (s, b)
                assert la['comm'] == o['comm'] and la['comp'] == o['comp'], (s, b)
                np.testing.assert_array_equal(la['trace_n_active'], o['trace_n_active'])
                np.testing.assert_array_equal(la['trace_tick'], o['trace_tick'])
    assert pool_entries <= 4 << 20
    rec = eng.job_records()
    n_checked = 0
    for (b, j), (k, nmw) in mounted.items():
        r = rec[b][j]
        if r['status'] not in (JS_RUNNING, JS_COMPLETED):
            continue
        o = want[k]
        assert r['jct'] == o['jct'] and r['comm'] == o['comm'] and r['comp'] == o['comp'], (b, j)
        assert r['util'] == oracle_lib.utilisation(o['trace_n_active'], o['trace_tick'], nmw, o['jct']), (b, j, nmw)
        n_checked += 1
    assert n_checked >= B
    eng.close()


@pytest.mark.gpu
@pytest.mark.parametrize('memo_mode', [1, 2])
def test_step_path_utilisation_with_varying_active_workers(memo_mode, eng_mod, oracle_lib):
    """The golden jobs keep one active-worker count on every busy tick, so a utilisation that reused one tick's
    n_active / n_mounted_workers for the others would still match them.  Here every job's busy ticks have 3-4 distinct
    active-worker counts.  Each job is mounted twice, one per step and job arrival, by B = 40 episodes on 1-4 extra
    workers: memo off, the second mount takes the hinted route; exact memo, one episode runs it and the step kernel
    recomputes the others' utilisation."""
    from ddls_b200.engine import JS_COMPLETED, JS_RUNNING, action_row
    ts = [_random_and_baseline()[k] for k in (2, 3, 12, 28, 32, 41)]
    want = [oracle_lib.run_lookahead(t) for t in ts]
    for o in want:
        busy = (o['trace_n_active'] > 0) & (o['trace_tick'] > 0)
        assert o['status'] == 0 and len(np.unique(o['trace_n_active'][busy])) >= 3
    order = list(range(len(ts))) * 2
    B, L = 40, len(order) + 1
    eng = eng_mod.RampEngine(n_episodes=B, n_cluster_workers=64, max_jobs=L, memo_mode=memo_mode, trace_cap=1 << 14)
    tids = [eng.register_template(t) for t in ts]
    assert all(eng.template_info(tid)['size_class'] == 2 for tid in tids)
    arr = np.zeros((B, L), dtype=eng_mod.ARRIVAL_DTYPE)
    arr['interarrival'] = 1e6                      # every job completes long before the next one arrives
    arr['interarrival'][:, -1] = np.inf
    eng.reset(arr)
    nmw = np.array([[ts[k].n_workers + (b % 4) for k in order] for b in range(B)])
    for s, k in enumerate(order):
        a = eng.make_actions()
        for b in range(B):
            action_row(a, b, tids[k], ts[k].mount)
            a['n_mounted_workers'][b] = nmw[b, s]
        eng.step(a, fuse_empty_steps=True)           # the job completes, then empty steps until the next one is queued
        eng.check_status()
        for b in range(B):
            la = eng.last_lookahead(b)
            assert la['jct'] == want[k]['jct'] and la['n_ticks'] == want[k]['n_ticks'], (s, b)
            np.testing.assert_array_equal(la['trace_n_active'], want[k]['trace_n_active'])
            np.testing.assert_array_equal(la['trace_tick'], want[k]['trace_tick'])
    rec = eng.job_records()
    for b in range(B):
        for s, k in enumerate(order):
            r, o = rec[b][s], want[k]
            assert r['status'] in (JS_RUNNING, JS_COMPLETED), (b, s)
            assert r['jct'] == o['jct'] and r['comm'] == o['comm'] and r['comp'] == o['comp'], (b, s)
            assert r['util'] == oracle_lib.utilisation(o['trace_n_active'], o['trace_tick'], int(nmw[b, s]), o['jct']), (b, s)
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# the tight build: two ring records per lane, the smallest shared-memory lists the small-frontier path allows, and a ledger
# lane slowed to 1 us per record, so the sim lane waits on a full ring and every non-trivial template spills every list
TIGHT_FLAGS = ['-DRAMP_T_RING=2', '-DRAMP_T_PUB=1', '-DRAMP_T_OCAP=2', '-DRAMP_T_FCAP=6', '-DRAMP_T_NFCAP=1',
               '-DRAMP_T_LEDGER_NS=1000']

TIGHT_SCRIPT = r'''
import sys
import numpy as np
sys.path[:0] = [{root!r}, {tests!r}]
from ddls_b200 import engine
engine.LIB_PATH = {lib!r}
engine.load_library()
from oracle import oracle
from golden_io import Golden
from conftest import golden_files
import test_gpu_thread_kernel as T
sets = [Golden(f).templates for f in golden_files() if f in T.RESIDENT and T.RESIDENT[f][0]]
sets += [T._random_and_baseline(), [c[1] for c in T.BOUNDARY]]
n = 0
for ts in sets:
    for mode in T.THREAD_MODES:
        for launch in ('first', 'hinted'):
            eng = T._engine(engine, mode, n_episodes=1, n_cluster_workers=64, max_jobs=1, trace_cap=1 << 16)
            tids = np.array([eng.register_template(t) for t in ts], dtype=np.int32)
            ids = np.repeat(tids, 2)
            if launch == 'hinted':
                eng.run_lookaheads(ids)
            res, _, tn, tt = eng.run_lookaheads(ids, want_trace=True)
            for k, t in enumerate(ts):
                o = oracle.run_lookahead(t)
                T._assert_equal_oracle(res, tn, tt, 2 * k, o)
                T._assert_equal_oracle(res, tn, tt, 2 * k + 1, o)
                n += 2
            eng.close()
print('tight ok', n)
'''


@pytest.mark.gpu
def test_tight_build_ring_backpressure_and_spills(eng_mod, oracle_lib):
    """The same kernel built with the tight capacities: golden, random, baseline and boundary sets, first launch and hinted,
    equal the oracle.  Built under build_variants/ (never over the normal library) and run in a subprocess, since the
    engine binding loads one library per process."""
    import time
    from ddls_b200 import build
    out = os.path.join(ROOT, 'build_variants', 'tight', 'libramp_b200.so')
    t0 = time.time()
    build.build(extra_flags=TIGHT_FLAGS, out=out)
    print(f'tight variant build: {time.time() - t0:.1f} s')
    code = TIGHT_SCRIPT.format(root=ROOT, tests=os.path.join(ROOT, 'tests'), lib=out)
    p = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
    assert 'tight ok' in p.stdout
