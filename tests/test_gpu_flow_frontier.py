"""Hinted thread-kernel launches on templates that stress its key-ordered ready-flow frontier, against the CPU oracle.

The kernel keeps the ready flows in descending key order: a completed class's flows are merged in, survivors are
compacted in order, and the small-frontier half takes the channel winners in one pass over that order
(tests/test_flow_frontier_model.py checks the rule on a model).  Here the templates are built so that the order is
exercised where it can break: equal keys on overlapping group sets (the bench's quotients split entries per channel group),
flows without a channel, classes completing while flows are still ready (merges into a non-empty frontier, with keys that
interleave), wide fans that carry a lookahead into the general half (more than 6 ready flows or 2 ready classes) and back,
zero-time flows and zero-cost ops.  Every lookahead runs twice, so the second, hinted launch is the one compared.
"""
import numpy as np
import pytest

import quotient_model as qm
from ddls_b200.quotient import quotient as native_quotient
from test_gpu_thread_kernel import FASTF, THREAD_MODES, _assert_equal_oracle, _engine, _job, resident_rule


def interleaved_merge_template():
    """Ops 0, 1, 2 on three workers finish at t = 1, 2, 3; each sends flows (long run times) to the sink on channels that
    overlap, with priorities that interleave across the three classes, so every completion after the first merges into
    a non-empty frontier.  Two flows have no channel, two have zero run time; op 3 costs nothing."""
    edges = []
    for src in range(3):
        for j in range(4):
            prio = 3 * j + src                                         # interleaved keys
            chan = None if (src, j) in ((0, 3), (2, 1)) else (src + j) % 3
            rt = 0.0 if (src, j) in ((1, 0), (2, 3)) else 4.0 + 0.5 * j + 0.125 * src
            edges.append((src, 4, rt, 1, chan, prio))
        edges.append((src, 3, 0.25 + 0.25 * src, 1, src % 3, 20 + src))
    edges.append((3, 4, 0.5, 1, 1, 30))
    return _job([1.0, 2.0, 3.0, 0.0, 0.5], [0, 1, 2, 0, 1], edges, 3, 3)


def bench_templates():
    from ddls_b200 import synth
    from ddls_b200.template_builder import RampShape, build_template
    return [build_template(synth.resnet_like_graph(), d, RampShape(4, 4, 4)) for d in (2, 4, 8, 16)]


def wide_fan_templates():
    """Random DAGs with many out-edges per op: frontiers beyond the small-frontier half in mid-lookahead."""
    from ddls_b200.template_builder import random_dag_template
    rng = np.random.default_rng(2024)
    return [random_dag_template(rng, int(n), avg_out=float(a), n_workers=int(w)) for n, a, w in
            zip(rng.integers(8, 60, size=24), rng.uniform(3.0, 9.0, size=24), rng.integers(1, 5, size=24))]


@pytest.mark.gpu
@pytest.mark.parametrize('mode', THREAD_MODES)
def test_hinted_key_ordered_frontier_vs_oracle(mode, oracle_lib):
    import torch
    assert torch.cuda.is_available(), 'this test needs a CUDA device'
    from ddls_b200 import engine
    engine.load_library()
    ts = [interleaved_merge_template()] + bench_templates() + wide_fan_templates()
    eng = _engine(engine, mode, n_episodes=1, n_cluster_workers=64, max_jobs=1, trace_cap=1 << 14)
    tids = np.array([eng.register_template(t) for t in ts], dtype=np.int32)
    ids = np.repeat(tids, 2)
    eng.run_lookaheads(ids)                                            # first launches: record the hints
    res, _, tn, tt = eng.run_lookaheads(ids, want_trace=True)          # hinted launches
    crossed = 0
    for k, t in enumerate(ts):
        q = native_quotient(t) if mode == 'thread' else qm.identity_quotient(t)
        if not resident_rule(t, q):
            continue
        o = oracle_lib.run_lookahead(t)
        _assert_equal_oracle(res, tn, tt, 2 * k, o)
        _assert_equal_oracle(res, tn, tt, 2 * k + 1, o)
        info = eng.template_info(int(tids[k]))
        assert info['size_class'] == 2 and (o['status'] != 0 or info['n_ticks'] == o['n_ticks']), k
        m = qm.run_lookahead_quotient(q)
        crossed += (m['max_f'] > FASTF or m['max_o'] > 2) and m['finished']
    assert crossed >= 4, crossed                                       # some lookaheads reach the general half
    eng.close()
